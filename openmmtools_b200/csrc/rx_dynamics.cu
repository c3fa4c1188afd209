// rx_dynamics.cu -- propagation (Langevin splitting dynamics) and the reduced-potential matrix.
//
// k_propagate   replaces MultiStateSampler._propagate_replicas (multistatesampler.py:1287-1337) ->
//               BaseIntegratorMove.apply (mcmc.py:668-776) -> LangevinIntegrator V/R/O substeps
//               (integrators.py:1404-1460): one CTA per replica, the replica lives in shared memory and
//               registers for all n_steps, one force evaluation per step (CustomIntegrator's lazy `f`).
// k_energy_rows replaces MultiStateSampler._compute_replica_energies (multistatesampler.py:1458-1494) ->
//               ThermodynamicState.reduced_potential_at_states (states.py:911-992): like the reference it
//               evaluates the lambda-independent groups once per configuration and only the
//               lambda-controlled pairs once per state (states.py:3649-3691).  All double precision.
// Energy function: alchemy/alchemy.py:1379-1388 (soft-core sterics), :1723-1750 / :1903-1919 (which pairs go
// to which force), testsystems.py:1956-1997 (switched LJ, cutoff-periodic).
#include "rx_internal.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;
#include <math.h>
#include <string.h>
#include <stdlib.h>

// ---------------------------------------------------------------------------------------------------
// Philox4x32-10 counter-based generator: noise is a pure function of (seed, iteration, replica, atom, step)
// ---------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ void philox_round(uint32_t &c0, uint32_t &c1, uint32_t &c2, uint32_t &c3,
                                                       uint32_t k0, uint32_t k1) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
    uint32_t c0 = ctr.x, c1 = ctr.y, c2 = ctr.z, c3 = ctr.w, k0 = key.x, k1 = key.y;
#pragma unroll
    for (int r = 0; r < 10; r++) {
        philox_round(c0, c1, c2, c3, k0, k1);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
}
// three standard normals from one Philox block (Box-Muller on words 0,1 and 2,3); fast-math intrinsics: the
// absolute error (~1e-6) is far below the float32 resolution of the velocity update it feeds
__device__ __forceinline__ float3 philox_normal3(uint4 r) {
    const float u1 = ((float)(r.x >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float u2 = ((float)(r.y >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float u3 = ((float)(r.z >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float u4 = ((float)(r.w >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float ra = sqrtf(-2.0f * __logf(u1)), rb = sqrtf(-2.0f * __logf(u3));
    float s1, c1;
    __sincosf(6.283185307179586f * u2, &s1, &c1);
    const float c2 = __cosf(6.283185307179586f * u4);
    return make_float3(ra * c1, ra * s1, rb * c2);
}

__device__ __forceinline__ float fast_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_rsqrt(float x) { float y; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// ---------------------------------------------------------------------------------------------------
// A Langevin splitting move: the launch's (DynParams::move), or one entry per thermodynamic state when the states carry
// different moves (multistatesampler.py:906-910: one MCMCMove per state; a replica is propagated with the move of the
// state it is in).  Built by make_move only.
struct MoveDev {
    float dt, a, b;             // timestep, O-step coefficients exp(-gamma h), sqrt(1-exp(-2 gamma h))
    int n_steps, n_prog, nV, nR, reassign;
    char prog[RX_MAX_PROGRAM];
    double dt_d, a_d, b_d;      // the same in f64 (the molecule kernel)
};

// A periodic box in float: the edges and their inverses.
struct BoxF { float Lx, Ly, Lz, iLx, iLy, iLz; };
__host__ __device__ __forceinline__ BoxF box_f(double X, double Y, double Z) {
    return {(float)X, (float)Y, (float)Z, (float)(1.0 / X), (float)(1.0 / Y), (float)(1.0 / Z)};
}

struct DynParams {
    int N, kind;
    BoxF box;                   // (NPT: each replica has its own, box[r])
    float rc2, rs2, rs, inv_w;  // cutoff^2, switch^2, switch, 1/(rc-rs)
    int use_switch, annihilate, c_is_6;
    float sc_c;                 // softcore_c
    int maxnb;                  // Verlet-list capacity per atom (0: all-pairs only)
    int sort_atoms;             // re-deal atoms to threads by neighbour count at every list build
    float rl2, rin2;            // (cutoff + skin_out)^2, (cutoff + skin_in)^2
    float half_in2, half_out2;  // (skin_in/2)^2, ((skin_out - skin_in)/2)^2
    MoveDev move;
};

struct PairLam { float la, ob; };

// Pair interaction in float: returns -dU/dr / r (so f_i += ret * (xi - xj)) and optionally the energy.
// One formula for every pair kind: plain LJ is the soft core with lambda^a = 1, alpha (1-lambda)^b = 0
// (x = (sigma/r)^6), so a warp never diverges on the pair kind.  Approximate reciprocals (1 ulp-class MUFU ops).
// C6: softcore_c == 6 (the reference default, alchemy.py:424); SW: the switching function is on.
template <bool C6, bool SW, bool ENERGY>
__device__ __forceinline__ float lj_pair_f(const DynParams &p, float r2, float sig, float eps, bool softcore,
                                           PairLam lam, float &energy) {
    const float la = softcore ? lam.la : 1.0f, ob = softcore ? lam.ob : 0.0f;
    const float inv_r2 = fast_rcp(r2);
    const float q = r2 * fast_rcp(sig * sig);
    float rsc, x, iD;
    if (C6) { rsc = q * q * q; iD = fast_rcp(ob + rsc); x = iD; }
    else { rsc = __powf(q, 0.5f * p.sc_c); const float D = ob + rsc; iD = fast_rcp(D); x = __powf(D, -6.0f / p.sc_c); }
    const float t4 = la * 4.0f * eps;
    const float tx = t4 * x;
    float e = tx * (x - 1.0f);
    // -dU/dr / r = t4 (2x-1) 6 x (r/sigma)^c / (D r^2)
    float fr = tx * (12.0f * x - 6.0f) * (rsc * iD) * inv_r2;
    if (SW && r2 > p.rs2) {
        const float rinv = fast_rsqrt(r2);
        const float r = r2 * rinv;
        const float t = (r - p.rs) * p.inv_w;
        const float t2 = t * t;
        const float S = 1.0f + t2 * t * (-10.0f + t * (15.0f - 6.0f * t));
        const float dS = t2 * (-30.0f + t * (60.0f - 30.0f * t)) * p.inv_w;
        fr = fr * S - e * dS * rinv;
        e *= S;
    }
    if (ENERGY) energy = e;
    return fr;
}

__device__ __forceinline__ double block_reduce_sum(double v, double *s_red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) s_red[w] = v;
    __syncthreads();
    double t = 0;
    if (threadIdx.x == 0) for (int q = 0; q < nw; q++) t += s_red[q];  // fixed order: deterministic
    return t;  // valid on thread 0
}

// Shared-memory accesses by 32-bit shared-space address: the generic-pointer path re-derives the CTA's shared window
// (S2R SR_CgaCtaId + LEA) inside the pair loop.
__device__ __forceinline__ float4 lds_f4(unsigned a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}
#define RX_MAX_ATOMS 1024      // atoms per block (one per thread); the shared-memory stride of the layout up to that size
#define RX_MAX_ATOMS_LJ 4096   // atoms per replica of the LJ kernels (k_propagate over a cluster of up to 8 blocks)
__device__ __forceinline__ float2 lds_f2(unsigned a) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ unsigned lds_u16(unsigned a) {
    unsigned short v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u16(unsigned a, unsigned v) {
    asm volatile("st.shared.u16 [%0], %1;" :: "r"(a), "h"((unsigned short)v) : "memory");
}

// Minimum image without the XU pipe: round-to-nearest-even of d/L through the 1.5*2^23 magic constant
// (|d/L| < 2^22), two FMA-pipe operations instead of FMUL + FRND.
__device__ __forceinline__ float min_image_f(float d, float L, float iL) {
    const float n = __fadd_rn(__fmaf_rn(d, iL, 12582912.0f), -12582912.0f);
    return __fmaf_rn(-L, n, d);
}
// The minimum image of the displacement (dx, dy, dz), in place; returns its square.
__device__ __forceinline__ float image_r2(const BoxF &b, float &dx, float &dy, float &dz) {
    dx = min_image_f(dx, b.Lx, b.iLx); dy = min_image_f(dy, b.Ly, b.iLy); dz = min_image_f(dz, b.Lz, b.iLz);
    return dx * dx + dy * dy + dz * dz;
}
// Wrap a position into the box (getState(enforcePeriodicBox=True), mcmc.py:731).
__device__ __forceinline__ void wrap_into(const BoxF &b, float &x, float &y, float &z) {
    x -= b.Lx * floorf(x * b.iLx); y -= b.Ly * floorf(y * b.iLy); z -= b.Lz * floorf(z * b.iLz);
}

// What the pair loop needs about atom i and its surroundings, gathered in registers before the loop.
struct PairCtx {
    BoxF box;
    float rc2;
    float x, y, z, sig_i, se_i;
    bool alch_i;
    PairLam lam;
    int reg_i;      // REG: region of atom i (0 environment, 1, 2)
    PairLam lam2;   // REG: the second region's lambda factors
};

// Pair rule of two alchemical regions (alchemy.py:1752-1777, 1903-1919 with two regions and no
// alchemical_regions_interactions): an environment-region pair is soft with that region's lambda, a same-region pair is
// soft only when that region annihilates (bit r-1 of `annihilate`), a pair across the regions has no interaction (`across`:
// the caller discards its terms, which are then exactly zero at any separation).  One formula for every pair kind.
__device__ __forceinline__ bool region_pair(int annihilate, int ri, int rj, PairLam lam2, PairLam &lam, bool &across) {
    const int rr = ri | rj;   // 0 environment, 1 or 2 one region, 3 across
    if (rr >= 2) lam = lam2;
    across = rr == 3;
    return ri != rj || (((annihilate << 1) >> ri) & 1);
}

// One candidate pair with atom j (position records at pos_base; parameter records par_off bytes further, or with P8
// 8-byte parameter records (sqrt_eps, alch) starting at the shared address par_off).  REG: the records carry region ids.
template <bool C6, bool SW, bool ENERGY, bool P8 = false, bool REG = false>
__device__ __forceinline__ void pair_term(const DynParams &p, const PairCtx &c, unsigned pos_base, int par_off, unsigned j,
                                          float &ax, float &ay, float &az, float &en) {
    const unsigned aj = pos_base + 16u * j;
    const float4 pj = lds_f4(aj);
    float dx = c.x - pj.x, dy = c.y - pj.y, dz = c.z - pj.z;
    const float r2 = image_r2(c.box, dx, dy, dz);
    if (r2 < c.rc2) {
        const float2 qj = lds_f2(P8 ? (unsigned)par_off + 8u * j : aj + (unsigned)par_off);
        bool soft, across = false;
        PairLam lam = c.lam;
        if constexpr (REG) {
            soft = region_pair(p.annihilate, c.reg_i, (int)qj.y, c.lam2, lam, across);
        } else {
            const bool alch_j = qj.y != 0.f;
            soft = (c.alch_i != alch_j) || (c.alch_i && alch_j && p.annihilate);
        }
        float e;
        float fr = lj_pair_f<C6, SW, ENERGY>(p, r2, 0.5f * (c.sig_i + pj.w), c.se_i * qj.x, soft, lam, e);
        if (REG && across) { fr = 0.f; e = 0.f; }
        ax += fr * dx; ay += fr * dy; az += fr * dz;
        if (ENERGY) en += 0.5f * e;
    }
}

// Force on one atom from the inner part of its neighbour list or, in the fallback, from all other atoms.
template <bool C6, bool SW, bool ENERGY, bool P8 = false, bool REG = false>
__device__ __forceinline__ void lj_forces(const DynParams &p, const PairCtx &c, unsigned pos_base, int par_off,
                                          unsigned nb_t, int N, int ncol, int a, bool use_list, int n_inner,
                                          float &fx, float &fy, float &fz, float &en) {
    float ax = 0.f, ay = 0.f, az = 0.f, e = 0.f;
    if (use_list) {
        const unsigned stride = 2u * (unsigned)ncol;
        unsigned q = nb_t;
        for (int n = 0; n < n_inner; n++, q += stride)
            pair_term<C6, SW, ENERGY, P8, REG>(p, c, pos_base, par_off, lds_u16(q), ax, ay, az, e);
    } else {
        for (int j = 0; j < N; j++)
            if (j != a) pair_term<C6, SW, ENERGY, P8, REG>(p, c, pos_base, par_off, (unsigned)j, ax, ay, az, e);
    }
    fx = ax; fy = ay; fz = az; en = e;
}

#define RX_SORT_BINS 128

// One CTA (or thread-block cluster) per owned replica, one atom per thread (N <= 1024 per block, N <= 4096 per replica).
//
// Neighbour search is a dual list held in shared memory, one column per thread:
//   outer list  every j with r < cutoff + skin_out when it was built (an all-pairs pass);
//   inner list  the leading n_inner entries of the column: the outer entries with r < cutoff + skin_in when the
//               column was last partitioned.  The force loop visits only these.
// The column is re-partitioned when some atom has moved more than skin_in/2 since the last partition, and the outer
// list is rebuilt when (checked at that moment) some atom has moved more than (skin_out - skin_in)/2 since the build,
// so that a pair missing from the outer list is still farther than cutoff + skin_in.
//
// Which atom a thread owns is re-decided at every outer build: atoms are dealt to threads in order of their inner
// neighbour count, so the lanes of a warp run pair loops of nearly equal length.  Per-atom results do not depend on
// the assignment (each atom sums its own list in list order, noise is keyed by atom id, the energy reductions run in
// atom order).
//
// Positions are double buffered: a force evaluation writes the moved positions into the buffer the previous
// evaluation did not read, and the displacement vote (__syncthreads_or) is the only barrier of the step.
// A replica may be split over a cluster of CL thread blocks (CL = 1, 2 or 4 up to 1024 atoms, chosen when there are fewer
// replicas than SMs; CL = 2, 4 or 8 above, where one block cannot hold the atoms):
// block q of the cluster owns the atoms [q Nq, (q+1) Nq), every block keeps ALL positions in its own shared memory -- a block
// writes the new positions of its atoms into every block's buffer through distributed shared memory -- and the step's only
// barrier becomes a cluster barrier.  The displacement votes are cluster wide, so the lists are rebuilt at the same steps and
// with the same contents as in one block: trajectories do not depend on CL (each atom sums its own list in list order, noise
// is keyed by atom id).
// PS: per-state moves (the move comes from `moves[state]` instead of `p.move`).
// COMPACT: the layout above 1024 atoms (DESIGN 4.2): position buffers strided by N instead of RX_MAX_ATOMS and 8-byte
// parameter records (sqrt_eps, alch) -- sigma rides in the position's w -- so that 4096 atoms leave room for a list.
// NPT: the box is the replica's (box[r], kept in f64 there) and a Monte Carlo barostat attempt opens every 25th step
// (rx_b200.h, rx_set_pressures); npt[state] = (pressure, dispersion coefficient), min_edge = twice the cutoff.
// REG: two alchemical regions (rx_set_alchemical_regions): the parameter records carry each atom's region id instead of the
// alchemical flag and the pair rule is region_pair's.
template <bool C6, bool SW, int CL, bool PS = false, bool COMPACT = false, bool NPT = false, bool REG = false>
__global__ void __launch_bounds__(1024) k_propagate(DynParams p, const float4 *__restrict__ atom,
                                                    const StateDev *__restrict__ states, const int *__restrict__ perm,
                                                    float4 *__restrict__ pos, float4 *__restrict__ vel, int k0,
                                                    uint2 key, uint32_t iteration,
                                                    double *__restrict__ pot, double *__restrict__ kin,
                                                    int *__restrict__ nan_flag, const int *__restrict__ only,
                                                    const MoveDev *__restrict__ moves, double4 *__restrict__ box,
                                                    rx_barostat_state *__restrict__ baro, const double2 *__restrict__ npt,
                                                    double min_edge) {
    extern __shared__ float4 s_dyn[];
    // (the whole cluster takes this exit together: `only` is indexed by replica)
    if (only && !only[k0 + blockIdx.x / CL]) return;   // a retry launch propagates the replicas that failed, nothing else
    // s_dyn[0..] / s_dyn[pos1..]: the two position buffers (pos1 = 2*MAX, or N when COMPACT)
    const int pos1 = COMPACT ? p.N : 2 * RX_MAX_ATOMS;
    float4 *s_par = s_dyn + RX_MAX_ATOMS;  // [RX_MAX_ATOMS] (sqrt_eps, alch, -, -)
    float2 *s_par8 = (float2 *)(s_dyn + 2 * p.N);                     // COMPACT: [N] (sqrt_eps, alch)
    float4 *s_ref = COMPACT ? s_dyn + (2 * p.N + (p.N + 1) / 2)      // [nthr] the thread's position at the last outer build
                            : s_dyn + 3 * RX_MAX_ATOMS;
    unsigned short *s_nb = (unsigned short *)(s_ref + blockDim.x);  // [maxnb][nthr] lists, slot-major (conflict free)
    __shared__ double s_red[32];
    __shared__ int s_vote[2];            // cluster-wide votes (alternating words)
    __shared__ double s_part[3 * (CL > 4 ? CL : 4)];   // per-block partial sums, gathered in block 0 of the cluster
    const int r = blockIdx.x / CL, q = blockIdx.x % CL, k = k0 + r, t = threadIdx.x, nthr = blockDim.x;
    const int Nq = (p.N + CL - 1) / CL, a_base = q * Nq;
    const int n_own = min(Nq, p.N - a_base);
    const bool active = t < n_own;   // threads beyond the block's atoms own none (they keep an id past the block's range)
    int a = a_base + t;              // the atom this thread owns
    unsigned vote_id = 0;
    if (t < 2) s_vote[t] = 0;
    // OR of `flag` over all threads of the cluster (of the block when CL == 1), doubling as the step's barrier
    auto cluster_or = [&](bool flag) -> bool {
        if (CL == 1) return __syncthreads_or(flag ? 1 : 0) != 0;
        vote_id++;
        int *word = &s_vote[vote_id & 1u];
        if (flag) {
            cg::cluster_group cl = cg::this_cluster();
#pragma unroll
            for (int c = 0; c < CL; c++) *cl.map_shared_rank(word, c) = (int)vote_id;   // every voter writes the same value
        }
        cg::this_cluster().sync();   // release / acquire: the positions and the votes written before it are visible
        return *(volatile int *)word == (int)vote_id;
    };
    const StateDev st = states[perm[k]];
    const PairLam lam = {(float)st.la, (float)st.ob};
    // the box the kernel computes in; NPT: the replica's (also kept in f64) and its barostat state
    BoxF bf = p.box;
    double bx = 0.0, by = 0.0, bz = 0.0;
    rx_barostat_state bs = {};
    double2 nst = {};
    if constexpr (NPT) {
        const double4 b4 = box[r];
        bx = b4.x; by = b4.y; bz = b4.z;
        bs = baro[r];
        nst = npt[perm[k]];
        bf = box_f(bx, by, bz);
    }
    // the move: the launch's, or the one of this replica's state
    const MoveDev &mv = PS ? moves[perm[k]] : p.move;
    const float m_a = mv.a, m_b = mv.b;   // (read once: the loop reads them under branches)
    const int m_steps = mv.n_steps, m_nprog = mv.n_prog;
    // (the program is interpreted: the compiler does not hoist these divisions out of the step loop; same values, same bits)
    const float h_V = mv.dt / (float)mv.nV, h_R = mv.dt / (float)mv.nR;
    float sig_i, se_i, inv_m, sigma_v;
    bool alch_i;
    int reg_i = 0;
    auto load_atom = [&]() {
        const float4 a4 = active ? atom[a] : make_float4(1.f, 0.f, 1.f, 0.f);
        sig_i = a4.x; se_i = a4.y; inv_m = a4.z; alch_i = a4.w != 0.f;
        if constexpr (REG) reg_i = (int)a4.w;
        sigma_v = sqrtf((float)st.kT * inv_m);  // sqrt(kT/m), integrators.py:1314
    };
    load_atom();
    float4 x4 = active ? pos[(size_t)r * p.N + a] : make_float4(0, 0, 0, 0);
    float4 v4 = active ? vel[(size_t)r * p.N + a] : make_float4(0, 0, 0, 0);
    float x = x4.x, y = x4.y, z = x4.z, vx = v4.x, vy = v4.y, vz = v4.z;
    if (mv.reassign && active) {  // context.setVelocitiesToTemperature, mcmc.py:711
        const float3 g = philox_normal3(philox4x32_10(make_uint4(a, 0x80000000u, k, iteration), key));
        vx = sigma_v * g.x; vy = sigma_v * g.y; vz = sigma_v * g.z;
    }
    for (int j = t; j < p.N; j += nthr) {   // parameter records of ALL atoms (the pair loop reads those of its partners)
        const float4 a4 = atom[j];
        const float tag = REG ? a4.w : (a4.w != 0.f ? 1.f : 0.f);
        if (COMPACT) s_par8[j] = make_float2(a4.y, tag);
        else s_par[j] = make_float4(a4.y, tag, 0.f, 0.f);
    }
    if (CL > 1) cg::this_cluster().sync();   // every block of the cluster is resident and has cleared its vote words
    float fx = 0, fy = 0, fz = 0;
    bool f_valid = false;
    const float hx0 = (float)st.ho_x0[0], hx1 = (float)st.ho_x0[1], hx2 = (float)st.ho_x0[2], hK = (float)st.ho_K;
    const bool lj = p.kind != RX_SYSTEM_HARMONIC;

    bool use_list = lj && p.maxnb > 0;
    bool have_list = false;        // an outer list exists
    bool built_once = false;       // NPT: an outer list was built in this launch (a volume move clears have_list only)
    int n_all = 0, n_inner = 0;
    float xi = x, yi = y, zi = z;  // position at the last partition
    int cur = 1;                   // position buffer of the latest force evaluation (0: s_dyn, 1: s_dyn + pos1)
    const unsigned dyn_base = (unsigned)__cvta_generic_to_shared(s_dyn);
    const unsigned nb_t = (unsigned)__cvta_generic_to_shared(s_nb + t);
    const unsigned stride = 2u * (unsigned)nthr;

    // Deal the atoms to the threads again, sorted by (inner neighbour count, atom's previous thread): a stable
    // counting sort through scratch space in the (dead) list area.
    auto reassign_atoms = [&](const float4 *s_pos) {
        const int nw = nthr >> 5, lane = t & 31, w = t >> 5;
        float4 *x_v = (float4 *)s_nb;                                // [nthr] velocities by atom id
        unsigned short *x_order = (unsigned short *)(x_v + nthr);    // [nthr] atom of each new thread
        unsigned short *x_cnt = x_order + nthr;                      // [nw][BINS] per-warp bin counts -> offsets
        unsigned short *x_base = x_cnt + nw * RX_SORT_BINS;          // [BINS] bin totals -> bases
        const int bin = active ? min(n_inner, RX_SORT_BINS - 2) : RX_SORT_BINS - 1;
        __syncthreads();  // every thread is done with its column (a partition may just have run)
        for (int q = t; q < nw * RX_SORT_BINS; q += nthr) x_cnt[q] = 0;
        x_v[a - a_base] = make_float4(vx, vy, vz, 0.f);
        __syncthreads();
        const unsigned m = __match_any_sync(0xffffffffu, bin);
        if (lane == __ffs(m) - 1) x_cnt[w * RX_SORT_BINS + bin] = (unsigned short)__popc(m);
        __syncthreads();
        for (int b = t; b < RX_SORT_BINS; b += nthr) {
            int run = 0;
            for (int q = 0; q < nw; q++) { const int c = x_cnt[q * RX_SORT_BINS + b]; x_cnt[q * RX_SORT_BINS + b] = (unsigned short)run; run += c; }
            x_base[b] = (unsigned short)run;
        }
        __syncthreads();
        if (t == 0) {
            int run = 0;
            for (int b = 0; b < RX_SORT_BINS; b++) { const int c = x_base[b]; x_base[b] = (unsigned short)run; run += c; }
        }
        __syncthreads();
        const int rank = x_base[bin] + x_cnt[w * RX_SORT_BINS + bin] + __popc(m & ((1u << lane) - 1u));
        x_order[rank] = (unsigned short)a;
        __syncthreads();
        a = x_order[t];
        const float4 vv = x_v[a - a_base];
        vx = vv.x; vy = vv.y; vz = vv.z;
        load_atom();
        if (active) { const float4 pa = s_pos[a]; x = pa.x; y = pa.y; z = pa.z; }
        __syncthreads();  // the scratch is dead: the list may be written
    };
    // Move the outer entries with r < cutoff + skin_in to the front of the column (every entry is tested once).
    auto partition = [&](const float4 *s_pos) {
        int lo = 0, hi = n_all - 1;
        if (active) {
            while (lo <= hi) {
                const unsigned ql = nb_t + (unsigned)lo * stride;
                const unsigned e = lds_u16(ql);
                const float4 pj = s_pos[e];
                float dx = x - pj.x, dy = y - pj.y, dz = z - pj.z;
                if (image_r2(bf, dx, dy, dz) < p.rin2) lo++;
                else {
                    const unsigned qh = nb_t + (unsigned)hi * stride;
                    sts_u16(ql, lds_u16(qh));
                    sts_u16(qh, e);
                    hi--;
                }
            }
        }
        n_inner = lo;
        xi = x; yi = y; zi = z;
    };
    auto build_outer = [&](const float4 *s_pos) {
        if (p.sort_atoms) reassign_atoms(s_pos);
        int cnt = 0;
        if (active) {
            for (int j = 0; j < p.N; j++) {
                const float4 pj = s_pos[j];
                float dx = x - pj.x, dy = y - pj.y, dz = z - pj.z;
                if (image_r2(bf, dx, dy, dz) < p.rl2 && j != a) {
                    if (cnt < p.maxnb) s_nb[cnt * nthr + t] = (unsigned short)j;
                    cnt++;
                }
            }
        }
        s_ref[t] = make_float4(x, y, z, 0.f);
        n_all = cnt;
        have_list = true;
        if constexpr (NPT) built_once = true;
        if (cluster_or(cnt > p.maxnb)) use_list = false;  // denser than the capacity: all-pairs from now on (the whole cluster)
    };
    // Make the list valid for the positions in buffer s_pos (all threads call this together).
    auto refresh_list = [&](const float4 *s_pos) {
        const float4 rf = s_ref[t];
        const float mx = x - rf.x, my = y - rf.y, mz = z - rf.z;
        const bool far = !have_list || (active && mx * mx + my * my + mz * mz > p.half_out2);
        if (cluster_or(far)) {
            bool first = !have_list;
            if constexpr (NPT) first = !built_once;   // (a rebuild after a volume move needs no counting pass)
            build_outer(s_pos);
            if (use_list) partition(s_pos);
            if (first && p.sort_atoms && use_list) {  // the first build only counted neighbours for the sort
                build_outer(s_pos);
                if (use_list) partition(s_pos);
            }
        } else {
            partition(s_pos);
        }
    };

    // The pair loop's context holds a second copy of bf, which the barostat refreshes with it: with bf alone (however it
    // reaches the pair loop) most NPT instantiations spill more (DESIGN 4.2).
    PairCtx pc;
    pc.box = bf; pc.rc2 = p.rc2; pc.lam = lam;
    if constexpr (REG) pc.lam2 = {(float)st.la2, (float)st.ob2};
    const int N = p.N;
    // Publish the current positions and make the neighbour list valid for them: one barrier unless a list is rebuilt.
    auto publish = [&]() {
        cur ^= 1;
        float4 *s_pos = s_dyn + (cur ? pos1 : 0);
        if (active) {
            const float4 me = make_float4(x, y, z, sig_i);
            if (CL == 1) s_pos[a] = me;
            else {
                cg::cluster_group cl = cg::this_cluster();
#pragma unroll
                for (int c = 0; c < CL; c++) cl.map_shared_rank(s_pos, c)[a] = me;
            }
        }
        const float mx = x - xi, my = y - yi, mz = z - zi;
        const bool moved = use_list && (!have_list || (active && mx * mx + my * my + mz * mz > p.half_in2));
        if (cluster_or(moved)) refresh_list(s_pos);
    };
    auto compute_forces = [&](bool want_energy, float &e_out) {
        if (!lj) {
            fx = -hK * (x - hx0); fy = -hK * (y - hx1); fz = -hK * (z - hx2);
            e_out = want_energy ? 0.5f * hK * ((x - hx0) * (x - hx0) + (y - hx1) * (y - hx1) + (z - hx2) * (z - hx2)) : 0.f;
            return;
        }
        if (!f_valid) publish();
        if (active) {
            pc.x = x; pc.y = y; pc.z = z; pc.sig_i = sig_i; pc.se_i = se_i; pc.alch_i = alch_i;
            if constexpr (REG) pc.reg_i = reg_i;
            const unsigned pos_base = dyn_base + (cur ? 16u * (unsigned)pos1 : 0u);
            // (COMPACT: the address of the 8-byte records; otherwise the offset from either buffer to the 16-byte records)
            const int par_off = COMPACT ? (int)(dyn_base + 32u * (unsigned)N) : (cur ? -16 * RX_MAX_ATOMS : 16 * RX_MAX_ATOMS);
            if (want_energy) lj_forces<C6, SW, true, COMPACT, REG>(p, pc, pos_base, par_off, nb_t, N, nthr, a, use_list, n_inner, fx, fy, fz, e_out);
            else lj_forces<C6, SW, false, COMPACT, REG>(p, pc, pos_base, par_off, nb_t, N, nthr, a, use_list, n_inner, fx, fy, fz, e_out);
        } else {
            fx = fy = fz = 0.f; e_out = 0.f;
        }
    };

    // ---- NPT: the Monte Carlo barostat (DESIGN 4.2) -------------------------------------------------------------
    // (the whole body is a discarded statement in the NVT instantiations, which compile exactly as without it)
    uint32_t n_baro = 0;   // attempts in this launch: the counter of the barostat's Philox stream
    auto barostat = [&]() {
        if constexpr (NPT) {
            auto cluster_sync = [&]() { if (CL == 1) __syncthreads(); else cg::this_cluster().sync(); };
            // Cluster-wide sum of the per-atom energies in fixed point (2^-24 kJ/mol): integer additions are associative, so the
            // total -- and every accept decision -- is the same bits in every block, at every cluster width and thread
            // assignment.  False in `fine` when some term is not finite or too large for the format (the move is then rejected).
            auto energy_sum = [&](float e, bool &fine) -> long long {
                unsigned long long *acc = (unsigned long long *)s_red;   // [0] sum, [1] terms out of range (in block 0)
                if (q == 0 && t < 2) acc[t] = 0ull;
                cluster_sync();
                const bool ok = !(fabsf(e) >= 67108864.0f) && !isnan(e);
                unsigned long long v = ok ? (unsigned long long)__double2ll_rn((double)e * 16777216.0) : 0ull, bad = ok ? 0ull : 1ull;
                for (int o = 16; o > 0; o >>= 1) { v += __shfl_xor_sync(0xffffffffu, v, o); bad += __shfl_xor_sync(0xffffffffu, bad, o); }
                unsigned long long *dst = acc;
                if (CL > 1) dst = cg::this_cluster().map_shared_rank(acc, 0);
                if ((t & 31) == 0) { atomicAdd(dst, v); if (bad) atomicAdd(dst + 1, bad); }
                cluster_sync();
                const long long total = (long long)dst[0];
                fine = dst[1] == 0ull;
                cluster_sync();   // every block has read the sums before they are cleared again
                return total;
            };
            auto set_box = [&](double X, double Y, double Z) { bf = box_f(X, Y, Z); pc.box = bf; };
            float e0;
            compute_forces(true, e0);   // (forces already valid come out the same bits: same list, same order)
            f_valid = true;
            bool fine0;
            const long long U0 = energy_sum(e0, fine0);
            const uint4 rr = philox4x32_10(make_uint4(n_baro++, 0xA0000000u, k, iteration), key);
            const double u1 = ((double)rr.x + 0.5) * 2.3283064365386963e-10, u2 = ((double)rr.y + 0.5) * 2.3283064365386963e-10;
            const double V = bx * by * bz, dV = bs.volume_scale * (2.0 * u1 - 1.0), V1 = V + dV;
            const double sc = V1 > 0.0 ? cbrt(V1 / V) : 0.0;
            bs.n_attempted++;
            if (fine0 && bx * sc >= min_edge && by * sc >= min_edge && bz * sc >= min_edge) {
                const int c_old = cur;   // the buffer holding the unscaled positions of every atom
                const float sf = (float)sc;
                x *= sf; y *= sf; z *= sf;
                set_box(bx * sc, by * sc, bz * sc);
                have_list = false;       // the list is rebuilt for the scaled box (and again after a rejection)
                f_valid = false;
                float e1;
                compute_forces(true, e1);
                f_valid = true;
                bool fine1;
                const long long U1 = energy_sum(e1, fine1);
                const double kT = st.kT;
                const double w = (double)(U1 - U0) * (1.0 / 16777216.0) + nst.y * (1.0 / V1 - 1.0 / V) + nst.x * dV -
                                 (double)p.N * kT * log(V1 / V);
                if (fine1 && (w <= 0.0 || u2 < exp(-w / kT))) {
                    bx *= sc; by *= sc; bz *= sc;
                    bs.n_accepted++;
                } else {
                    // the thread's atom may have changed in the rebuild: its unscaled position comes from the old buffer
                    if (active) { const float4 o = (s_dyn + (c_old ? pos1 : 0))[a]; x = o.x; y = o.y; z = o.z; }
                    set_box(bx, by, bz);
                    have_list = false;
                    f_valid = false;
                }
            }
            if (bs.n_attempted >= 10) {
                if (bs.n_accepted < 0.25 * bs.n_attempted) { bs.volume_scale /= 1.1; bs.n_attempted = bs.n_accepted = 0; }
                else if (bs.n_accepted > 0.75 * bs.n_attempted) {
                    bs.volume_scale = fmin(bs.volume_scale * 1.1, 0.3 * V);
                    bs.n_attempted = bs.n_accepted = 0;
                }
            }
        }
    };

    uint32_t ocount = 0;
    float dummy;
    for (int s = 0; s < m_steps; s++) {
        if constexpr (NPT) { if (++bs.step >= 25) { bs.step = 0; barostat(); } }
        for (int q = 0; q < m_nprog; q++) {
            const char op = mv.prog[q];
            if (op == 'V') {
                if (!f_valid) { compute_forces(false, dummy); f_valid = true; }
                const float h = h_V;
                vx += h * fx * inv_m; vy += h * fy * inv_m; vz += h * fz * inv_m;
            } else if (op == 'R') {
                const float h = h_R;
                x += h * vx; y += h * vy; z += h * vz;
                f_valid = false;
            } else {  // 'O'
                const float3 g = philox_normal3(philox4x32_10(make_uint4(a, ocount, k, iteration), key));
                ocount++;
                vx = m_a * vx + m_b * sigma_v * g.x;
                vy = m_a * vy + m_b * sigma_v * g.y;
                vz = m_a * vz + m_b * sigma_v * g.z;
            }
        }
    }
    // potential (in the replica's current state) and kinetic energy, SamplerState.potential_energy/kinetic_energy;
    // summed in atom order whatever the thread assignment is
    float e_i = 0;
    compute_forces(true, e_i);
    __syncthreads();  // the list is dead from here: its area carries the per-atom terms
    double2 *x_e = (double2 *)s_nb;
    x_e[a - a_base] = make_double2((double)e_i, active ? 0.5 * (double)(vx * vx + vy * vy + vz * vz) / (double)inv_m : 0.0);
    __syncthreads();
    const double2 et = x_e[t];
    double U = block_reduce_sum(t < n_own ? et.x : 0.0, s_red);
    double KE = block_reduce_sum(t < n_own ? et.y : 0.0, s_red);
    const bool bad = active && !(isfinite(x) && isfinite(y) && isfinite(z) && isfinite(vx) && isfinite(vy) && isfinite(vz));
    int any_bad = __syncthreads_or(bad ? 1 : 0);
    if (CL > 1) {   // block 0 of the cluster adds the partial sums in block order
        cg::cluster_group cl = cg::this_cluster();
        if (t == 0) {
            double *dst = cl.map_shared_rank(s_part, 0);
            dst[3 * q] = U; dst[3 * q + 1] = KE; dst[3 * q + 2] = any_bad ? 1.0 : 0.0;
        }
        cl.sync();
        if (q == 0 && t == 0) {
            U = 0; KE = 0; any_bad = 0;
            for (int c = 0; c < CL; c++) { U += s_part[3 * c]; KE += s_part[3 * c + 1]; any_bad |= s_part[3 * c + 2] != 0.0; }
        }
    }
    if (t == 0 && q == 0) {
        if constexpr (NPT) {
            pot[k] = U + st.offset + nst.y / (bx * by * bz);
            box[r] = make_double4(bx, by, bz, 0.0);
            baro[r] = bs;
        } else {
            pot[k] = U + st.offset;
        }
        kin[k] = KE;
        nan_flag[k] = (any_bad || !isfinite(U)) ? 1 : 0;
    }
    if (active) {
        if (lj) wrap_into(bf, x, y, z);
        pos[(size_t)r * p.N + a] = make_float4(x, y, z, 0.f);
        vel[(size_t)r * p.N + a] = make_float4(vx, vy, vz, 0.f);
    }
    if (CL > 1) cg::this_cluster().sync();   // no block leaves while another may still write into its shared memory
}

__global__ void k_randomize_velocities(int N, const float4 *__restrict__ atom, const StateDev *__restrict__ states,
                                       const int *__restrict__ perm, float4 *__restrict__ vel, int k0, uint2 key,
                                       uint32_t stream_id) {
    const int r = blockIdx.x, k = k0 + r;
    const StateDev st = states[perm[k]];
    for (int t = threadIdx.x; t < N; t += blockDim.x) {
        const float sv = sqrtf((float)st.kT * atom[t].z);
        const float3 g = philox_normal3(philox4x32_10(make_uint4(t, 0xC0000000u, k, stream_id), key));
        vel[(size_t)r * N + t] = make_float4(sv * g.x, sv * g.y, sv * g.z, 0.f);
    }
}

// ---------------------------------------------------------------------------------------------------
// Energy rows, double precision.
// ---------------------------------------------------------------------------------------------------
struct EnParams {
    int N, M, kind, n_alch;
    double Lx, Ly, Lz;
    double rc2, rs, rc, inv_w;
    int use_switch, annihilate, c_is_6;
    double sc_c;
    int pair_cap;
};

__device__ __forceinline__ double min_image_d(double d, double L) { return d - L * rint(d / L); }
__device__ __forceinline__ double switch_d(const EnParams &p, double r) {
    if (!p.use_switch || r <= p.rs) return 1.0;
    const double t = (r - p.rs) * p.inv_w;
    return 1.0 + t * t * t * (-10.0 + t * (15.0 - 6.0 * t));
}

// NPT: the replica's box from box[r], and u[k][l] gains beta_l (c_l / V_k + p_l V_k), npt[l] = (p_l, c_l).
// REG: two alchemical regions (atom_d[i].w is the region id; the pair rule of region_pair).  A lambda-controlled pair record
// carries its region in the sign of its first word (negative: region 2; the word, (r/sigma)^c, is > 0).
template <bool NPT = false, bool REG = false>
__global__ void __launch_bounds__(512) k_energy_rows(EnParams p, const double4 *__restrict__ atom_d,
                                                     const int *__restrict__ alch_list,
                                                     const StateDev *__restrict__ states,
                                                     const float4 *__restrict__ pos, int k0, double2 *__restrict__ pairs,
                                                     double *__restrict__ u, int *__restrict__ err,
                                                     const double4 *__restrict__ box, const double2 *__restrict__ npt) {
    extern __shared__ double s_en[];
    double *sx = s_en, *sy = s_en + p.N, *sz = s_en + 2 * p.N;
    __shared__ double s_red[32];
    __shared__ int s_scan[32];
    __shared__ double s_U0;
    __shared__ int s_npairs;
    const int r = blockIdx.x, k = k0 + r, t = threadIdx.x, nt = blockDim.x;
    if constexpr (NPT) { const double4 b = box[r]; p.Lx = b.x; p.Ly = b.y; p.Lz = b.z; }
    for (int q = t; q < p.N; q += nt) {
        const float4 x4 = pos[(size_t)r * p.N + q];
        sx[q] = (double)x4.x; sy[q] = (double)x4.y; sz[q] = (double)x4.z;
    }
    __syncthreads();
    double U0 = 0.0;
    if (p.kind == RX_SYSTEM_HARMONIC) {
        // u[k,l] = beta_l (sum_i K_l/2 |x_i - x0_l|^2 + offset_l)
        for (int l = t; l < p.M; l += nt) {
            const StateDev st = states[l];
            double U = 0;
            for (int i = 0; i < p.N; i++) {
                const double dx = sx[i] - st.ho_x0[0], dy = sy[i] - st.ho_x0[1], dz = sz[i] - st.ho_x0[2];
                U += 0.5 * st.ho_K * (dx * dx + dy * dy + dz * dz);
            }
            u[(size_t)k * p.M + l] = st.beta * (U + st.offset);
        }
        return;
    }
    // ---- phase 1: lambda-independent pairs (E-E, and A-A when not annihilating), half shell: i with i+1..i+N/2
    const int half = p.N / 2;
    for (int i = t; i < p.N; i += nt) {
        const double4 ai = atom_d[i];
        const bool alch_i = ai.w != 0.0;
        for (int d = 1; d <= half; d++) {
            if ((p.N % 2 == 0) && d == half && i >= half) break;  // the antipodal pair is counted once
            int j = i + d; if (j >= p.N) j -= p.N;
            const double4 aj = atom_d[j];
            const bool alch_j = aj.w != 0.0;
            bool soft;
            if constexpr (REG) {   // lambda-controlled or across the regions: not here
                const int ri = (int)ai.w, rj = (int)aj.w;
                soft = ri != rj || (((p.annihilate << 1) >> ri) & 1);
            } else {
                soft = (alch_i != alch_j) || (alch_i && alch_j && p.annihilate);
            }
            if (soft) continue;
            const double dx = min_image_d(sx[i] - sx[j], p.Lx), dy = min_image_d(sy[i] - sy[j], p.Ly),
                         dz = min_image_d(sz[i] - sz[j], p.Lz);
            const double r2 = dx * dx + dy * dy + dz * dz;
            if (r2 >= p.rc2) continue;
            const double sig = 0.5 * (ai.x + aj.x), eps = sqrt(ai.y * aj.y);
            const double s2 = sig * sig / r2, s6 = s2 * s2 * s2;
            U0 += 4.0 * eps * (s6 * s6 - s6) * switch_d(p, sqrt(r2));
        }
    }
    const double U0_tot = block_reduce_sum(U0, s_red);
    if (t == 0) s_U0 = U0_tot;
    // ---- phase 2: lambda-controlled pairs (alchemical atom a) x (atom j), deterministic order by a stable scan
    double2 *my_pairs = pairs + (size_t)r * p.pair_cap;
    int total = 0;
    for (int pass = 0; pass < 2; pass++) {
        int cnt = 0, base = 0;
        if (pass == 1) {
            // exclusive scan of per-thread counts (warp shuffle + warp totals)
            const int lane = t & 31, w = t >> 5, nw = (nt + 31) >> 5;
            int incl = total;  // `total` holds this thread's count from pass 0
            for (int o = 1; o < 32; o <<= 1) { int n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
            if (lane == 31) s_scan[w] = incl;
            __syncthreads();
            int woff = 0;
            for (int q = 0; q < w; q++) woff += s_scan[q];
            base = woff + incl - total;
            if (t == nt - 1) s_npairs = base + total;
            (void)nw;
        }
        for (int ai_ = 0; ai_ < p.n_alch; ai_++) {
            const int a = alch_list[ai_];
            const double4 pa = atom_d[a];
            for (int j = t; j < p.N; j += nt) {
                if (j == a) continue;
                const double4 pj = atom_d[j];
                const bool alch_j = pj.w != 0.0;
                if constexpr (REG) {   // same region: only when that region annihilates, counted once; across: never
                    if (alch_j && (pj.w != pa.w || !(((p.annihilate << 1) >> (int)pa.w) & 1) || j < a)) continue;
                } else {
                    if (alch_j && (!p.annihilate || j < a)) continue;  // A-A: only when annihilating, counted once
                }
                const double dx = min_image_d(sx[a] - sx[j], p.Lx), dy = min_image_d(sy[a] - sy[j], p.Ly),
                             dz = min_image_d(sz[a] - sz[j], p.Lz);
                const double r2 = dx * dx + dy * dy + dz * dz;
                if (r2 >= p.rc2) continue;
                if (pass == 1) {
                    const int slot = base + cnt;
                    if (slot < p.pair_cap) {
                        const double sig = 0.5 * (pa.x + pj.x), eps = sqrt(pa.y * pj.y);
                        const double q = r2 / (sig * sig);
                        const double rsc = p.c_is_6 ? q * q * q : pow(q, 0.5 * p.sc_c);
                        my_pairs[slot] = make_double2(REG && pa.w == 2.0 ? -rsc : rsc, 4.0 * eps * switch_d(p, sqrt(r2)));
                    }
                }
                cnt++;
            }
        }
        if (pass == 0) total = cnt;
    }
    __syncthreads();
    int npairs = s_npairs;
    if (npairs > p.pair_cap) { if (t == 0) atomicExch(err, RX_ERR_CAPACITY); npairs = p.pair_cap; }
    // ---- phase 3: one state per thread, pairs summed in list order
    const double U0s = s_U0;
    for (int l = t; l < p.M; l += nt) {
        const StateDev st = states[l];
        double Ua = 0.0;
        for (int q = 0; q < npairs; q++) {
            const double2 pr = my_pairs[q];
            if constexpr (REG) {
                const bool second = pr.x < 0.0;
                const double D = (second ? st.ob2 : st.ob) + fabs(pr.x);
                const double x = p.c_is_6 ? 1.0 / D : pow(D, -6.0 / p.sc_c);
                Ua += (second ? st.la2 : st.la) * pr.y * x * (x - 1.0);
            } else {
                const double D = st.ob + pr.x;
                const double x = p.c_is_6 ? 1.0 / D : pow(D, -6.0 / p.sc_c);
                Ua += st.la * pr.y * x * (x - 1.0);
            }
        }
        if constexpr (NPT) {
            const double V = p.Lx * p.Ly * p.Lz;
            const double2 pc = npt[l];
            u[(size_t)k * p.M + l] = st.beta * (U0s + Ua + st.offset + pc.y / V + pc.x * V);
        } else {
            u[(size_t)k * p.M + l] = st.beta * (U0s + Ua + st.offset);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// host <-> device conversions at the boundary (double xyz <-> float4)
// ---------------------------------------------------------------------------------------------------
__global__ void k_pack(const double *__restrict__ in, float4 *__restrict__ out, long long n) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i < n) out[i] = make_float4((float)in[3 * i], (float)in[3 * i + 1], (float)in[3 * i + 2], 0.f);
}
__global__ void k_unpack(const float4 *__restrict__ in, double *__restrict__ out, long long n, int wrap, double Lx,
                         double Ly, double Lz) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 v = in[i];
    double x = v.x, y = v.y, z = v.z;
    if (wrap) { x -= Lx * floor(x / Lx); y -= Ly * floor(y / Ly); z -= Lz * floor(z / Lz); }
    out[3 * i] = x; out[3 * i + 1] = y; out[3 * i + 2] = z;
}

int rxi_convert_in(rx_engine *h, float4 *dst, int first_local, int count, const double *host_xyz, bool) {
    const long long n = (long long)count * h->cfg.n_atoms;
    if (n == 0) return RX_OK;
    if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) {   // the state of a molecule is kept in f64: a plain copy
        double *d = (double *)dst + (size_t)first_local * h->cfg.n_atoms * 3;
        RX_CHECK_CUDA(h, cudaMemcpyAsync(d, host_xyz, n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
        RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
        return RX_OK;
    }
    const double *src = host_xyz;
    if (!rxi_is_pinned(h, host_xyz, n * 3 * sizeof(double))) {   // pageable caller memory goes through the pinned staging buffer
        memcpy(h->h_io, host_xyz, n * 3 * sizeof(double));
        src = h->h_io;
    }
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_io, src, n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    k_pack<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(h->d_io, dst + (size_t)first_local * h->cfg.n_atoms, n);
    RX_CHECK_CUDA(h, cudaGetLastError());
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return RX_OK;
}

int rxi_convert_out(rx_engine *h, const float4 *src, int first_local, int count, double *host_xyz, bool wrap) {
    const long long n = (long long)count * h->cfg.n_atoms;
    if (n == 0) return RX_OK;
    if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) {
        const double *d = (const double *)src + (size_t)first_local * h->cfg.n_atoms * 3;
        RX_CHECK_CUDA(h, cudaMemcpyAsync(host_xyz, d, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
        RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
        return RX_OK;
    }
    k_unpack<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(src + (size_t)first_local * h->cfg.n_atoms, h->d_io, n,
                                                                 wrap ? 1 : 0, h->cfg.box[0], h->cfg.box[1], h->cfg.box[2]);
    RX_CHECK_CUDA(h, cudaGetLastError());
    const bool direct = rxi_is_pinned(h, host_xyz, n * 3 * sizeof(double));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(direct ? host_xyz : h->h_io, h->d_io, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (!direct) memcpy(host_xyz, h->h_io, n * 3 * sizeof(double));
    return RX_OK;
}

#include "rx_molecule.cuh"

// A block may take 48 KB of shared memory, static and dynamic together, unless the kernel has opted in to more (up to
// cudaDevAttrMaxSharedMemoryPerBlockOptin, which mol_check_shared checks).  The molecule's tables grow with its terms, the
// energy kernel's coordinates with the atoms (48 KB of them at 2048 atoms, over the limit with its static arrays).
static int smem_opt_in(rx_engine *h, const void *kern, int dyn) {
    cudaFuncAttributes fa;
    RX_CHECK_CUDA(h, cudaFuncGetAttributes(&fa, kern));
    if (fa.sharedSizeBytes + (size_t)dyn > 48 * 1024)
        RX_CHECK_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
    return RX_OK;
}

// The dynamic shared memory of the molecule kernels (mol_gb_at): k_propagate_mol's (f32) or the others'; g: the GB kernels'.
static int mol_dyn_bytes(const MolDev &m, const MolGB *g, bool f32) { return mol_gb_at(m, f32) + (g ? g->prop_bytes : 0); }

// ---------------------------------------------------------------------------------------------------
// The move of a splitting program (V, R, O substeps) run n_steps times with timestep dt and friction gamma.
static MoveDev make_move(double dt, double gamma, int n_steps, const char *program, int reassign) {
    MoveDev d;
    memset(&d, 0, sizeof(d));
    int n = 0, nV = 0, nR = 0, nO = 0;
    for (const char *q = program; *q; q++, n++) { if (*q == 'V') nV++; else if (*q == 'R') nR++; else nO++; d.prog[n] = *q; }
    d.n_prog = n; d.nV = nV; d.nR = nR;
    d.dt = (float)dt; d.n_steps = n_steps; d.reassign = reassign;
    const double hO = dt / (nO > 0 ? nO : 1);   // integrators.py:1141-1146
    d.dt_d = dt; d.a_d = exp(-gamma * hO); d.b_d = sqrt(1.0 - exp(-2.0 * gamma * hO));
    d.a = (float)d.a_d; d.b = (float)d.b_d;
    return d;
}

static int fill_dyn(rx_engine *h, DynParams &p, int reassign) {
    const rx_config &c = h->cfg;
    memset(&p, 0, sizeof(p));
    p.N = c.n_atoms; p.kind = c.system_kind;
    p.box = box_f(c.box[0], c.box[1], c.box[2]);
    p.rc2 = (float)(c.r_cutoff * c.r_cutoff); p.rs2 = (float)(c.r_switch * c.r_switch); p.rs = (float)c.r_switch;
    p.inv_w = (float)(1.0 / (c.r_cutoff - c.r_switch));
    p.use_switch = c.use_switch; p.annihilate = h->two_regions ? h->annihilate_mask : c.annihilate_sterics;
    p.c_is_6 = (c.softcore_c == 6.0); p.sc_c = (float)c.softcore_c;
    p.maxnb = 0; p.sort_atoms = 0; p.rl2 = p.rin2 = p.rc2; p.half_in2 = p.half_out2 = 0.f;
    p.move = make_move(h->dt, h->gamma, h->n_steps, h->program, reassign);
    return RX_OK;
}

// The per-state move table (rx_set_state_integrator), uploaded when it changed.
int rxi_upload_state_moves(rx_engine *h) {
    if (!h->state_moves_dirty) return RX_OK;
    const int M = h->cfg.n_states;
    std::vector<MoveDev> tab((size_t)M);
    for (int l = 0; l < M; l++) {
        const rx_state_move &m = h->state_moves[(size_t)l];
        tab[(size_t)l] = make_move(m.dt, m.gamma, m.n_steps, m.program, m.reassign);
    }
    if (!h->d_moves) RX_CHECK_CUDA(h, cudaMalloc(&h->d_moves, sizeof(MoveDev) * (size_t)M));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_moves, tab.data(), sizeof(MoveDev) * (size_t)M, cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));   // (tab is a stack object)
    h->state_moves_dirty = false;
    return RX_OK;
}

// ---------------------------------------------------------------------------------------------------
// Launch plan of k_propagate: host arithmetic only (rx_plan_propagate exports it, so that it can be checked without a GPU).
// ---------------------------------------------------------------------------------------------------
#define RX_PROP_STATIC_SMEM 1024   // bound on k_propagate's static shared memory (s_red, s_vote, s_part: under 0.5 KB)
#define RX_MIN_LIST_CAP 48         // list entries per atom every cluster chosen above 1024 atoms holds (DESIGN 4.2)

// Dual neighbour list: outer skin 0.40 nm (at 300 K and 10/ps friction the all-pairs build usually lasts a whole 500-step
// launch), inner skin 0.05 nm (a re-partition of the column about every 25 steps; both tuned on the 512-atom fluid, see
// profiles/prop_r1_v6.summary.txt).  The outer radius is clipped to half the shortest box edge.
struct ListGeom { bool on; double rl, skin_in, eff_out; };
static ListGeom list_geometry(const rx_propagate_query *q) {
    ListGeom g = {false, 0.0, 0.0, 0.0};
    if (q->system_kind != RX_SYSTEM_LJ_ALCH || q->n_atoms < 64 || q->no_list) return g;
    const double skin_out = q->skin_out >= 0 ? q->skin_out : 0.40;
    double skin_in = q->skin_in >= 0 ? q->skin_in : 0.05;
    double rl = q->r_cutoff + skin_out;
    for (int d = 0; d < 3; d++) if (rl > 0.5 * q->box[d]) rl = 0.5 * q->box[d];
    const double eff_out = rl - q->r_cutoff;
    if (skin_in > eff_out / 3.0) skin_in = eff_out / 3.0;
    g.on = eff_out > 0.03; g.rl = rl; g.skin_in = skin_in; g.eff_out = eff_out;
    return g;
}

// Threads, list capacity, sort flag and dynamic shared memory of N atoms over `cl` blocks.  The list capacity comes from
// the shared-memory budget: up to 1024 atoms two CTAs per SM up to 512 threads (112 KB each), 200 KB above; the compact
// layout takes the device's opt-in limit.  Denser systems fall back to all-pairs in the kernel.  False: the atoms alone
// do not fit in the compact budget.
static bool plan_at(int N, int cl, bool compact, const ListGeom &g, size_t compact_budget, bool no_sort, rx_propagate_plan *o) {
    memset(o, 0, sizeof(*o));
    const int n_per = (N + cl - 1) / cl;
    const int threads = ((n_per + 31) / 32) * 32;
    // shared memory: two position buffers + the parameter records + per-thread reference positions + the list area
    // (compact: 16 + 16 + 8 bytes per atom, rounded up to 16 bytes; otherwise 3 x 16 bytes x RX_MAX_ATOMS)
    const size_t atoms_bytes = (compact ? ((size_t)40 * N + 15) / 16 * 16 : (size_t)3 * RX_MAX_ATOMS * sizeof(float4)) +
                               (size_t)threads * sizeof(float4);
    size_t area = (size_t)threads * sizeof(double2);  // the list area doubles as scratch for the final reductions
    if (g.on) {
        const size_t budget = compact ? compact_budget : (size_t)(threads > 512 ? 200 : 112) * 1024;
        int cap = budget > atoms_bytes ? (int)((budget - atoms_bytes) / ((size_t)threads * sizeof(unsigned short))) : 0;
        if (cap > 128) cap = 128;
        if (cap >= 8) {
            o->list_capacity = cap;
            const size_t list_bytes = (((size_t)cap * threads * sizeof(unsigned short)) + 15) / 16 * 16;
            // scratch of the atom re-assignment: velocities, order, per-warp bin counts, bin bases
            const size_t sort_bytes = (size_t)threads * (sizeof(float4) + 2) + (size_t)(threads / 32 + 1) * RX_SORT_BINS * 2;
            o->sort_atoms = (list_bytes >= sort_bytes && !no_sort) ? 1 : 0;
            if (list_bytes > area) area = list_bytes;
        }
    }
    o->cluster = cl;
    o->threads = threads;
    o->compact = compact ? 1 : 0;
    o->smem_bytes = (int64_t)(atoms_bytes + area);
    return !compact || atoms_bytes + area <= compact_budget;
}

int rxi_plan_propagate(const rx_propagate_query *q, rx_propagate_plan *o, std::string &err) {
    memset(o, 0, sizeof(*o));
    const int N = q->n_atoms;
    const bool lj = q->system_kind == RX_SYSTEM_LJ_ALCH;
    if (!lj && q->system_kind != RX_SYSTEM_HARMONIC) { err = "rx_plan_propagate: LJ and harmonic systems only"; return RX_ERR_INVALID; }
    if (N < 1 || q->kloc < 0 || q->n_sm < 1) { err = "rx_plan_propagate: need n_atoms >= 1, kloc >= 0, n_sm >= 1"; return RX_ERR_INVALID; }
    if (!lj && N > RX_MAX_ATOMS) {
        err = "rx_propagate: more than 1024 atoms per replica of a harmonic system is not supported";
        return RX_ERR_UNSUPPORTED;
    }
    if (N > RX_MAX_ATOMS_LJ) {
        err = "rx_propagate: more than 4096 atoms per replica is not supported (every block of a replica's cluster holds "
              "all of its positions in shared memory)";
        return RX_ERR_UNSUPPORTED;
    }
    const ListGeom g = list_geometry(q);
    if (N <= RX_MAX_ATOMS) {
        // Blocks per replica (a thread-block cluster; RX_CLUSTER = 1 | 2 | 4 overrides).  A block of 128 threads leaves ONE
        // warp per scheduler, which runs the step's
        // ~1100 dependent instructions no faster than four warps sharing a scheduler do: the split only pays for the few
        // replicas that would otherwise leave three quarters of the GPU idle, so that is the only case it is chosen for.
        int cl = 1;
        if (lj && N >= 256) {
            if (q->kloc * 4 <= q->n_sm) cl = 4;
            if (q->cluster == 1 || q->cluster == 2 || q->cluster == 4) cl = q->cluster;
        }
        if (q->per_state) cl = 1;
        plan_at(N, cl, false, g, 0, q->no_sort, o);
        return RX_OK;
    }
    // Above 1024 atoms a replica needs CL >= N/1024 blocks.  The smallest CL of 2, 4, 8 whose blocks hold the atoms and a
    // list of at least RX_MIN_LIST_CAP entries; widened to 4 or 8 when the replicas leave SMs idle (kloc CL <= #SMs).
    // RX_CLUSTER = 2 | 4 | 8 overrides when that CL can hold the atoms and such a list.
    const size_t budget = q->smem_optin > RX_PROP_STATIC_SMEM ? (size_t)q->smem_optin - RX_PROP_STATIC_SMEM : 0;
    rx_propagate_plan tmp;
    auto feasible = [&](int cl) {
        return cl * RX_MAX_ATOMS >= N && plan_at(N, cl, true, g, budget, q->no_sort, &tmp) &&
               (!g.on || tmp.list_capacity >= RX_MIN_LIST_CAP);
    };
    int cl = 0;
    for (int c = 2; c <= 8 && !cl; c *= 2) if (feasible(c)) cl = c;
    if (!cl) {
        err = "rx_propagate: " + std::to_string(N) + " atoms per replica do not fit in a cluster of up to 8 blocks with " +
              std::to_string(q->smem_optin) + " bytes of shared memory each";
        return RX_ERR_UNSUPPORTED;
    }
    for (int c = 8; c > cl; c /= 2)
        if ((long long)q->kloc * c <= q->n_sm && feasible(c)) { cl = c; break; }
    if ((q->cluster == 2 || q->cluster == 4 || q->cluster == 8) && feasible(q->cluster)) cl = q->cluster;
    plan_at(N, cl, true, g, budget, q->no_sort, o);
    return RX_OK;
}

// ---------------------------------------------------------------------------------------------------
// Launch tables: runtime choices to template arguments, over the instantiations that exist and no others.
// ---------------------------------------------------------------------------------------------------
// f(std::true_type) or f(std::false_type): a runtime flag as a template argument.
template <typename F> static auto with_flag(bool b, F &&f) { return b ? f(std::true_type{}) : f(std::false_type{}); }

// Launch one instantiation; opt_in: first allow it lc.dynamicSmemBytes of dynamic shared memory (above the 48 KB default).
template <typename... P, typename... A>
static int launch_kernel(rx_engine *h, const cudaLaunchConfig_t &lc, bool opt_in, void (*kern)(P...), A... args) {
    if (opt_in)
        RX_CHECK_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lc.dynamicSmemBytes));
    RX_CHECK_CUDA(h, cudaLaunchKernelEx(&lc, kern, args...));
    return RX_OK;
}

// The (CL, PS, COMPACT) layouts of k_propagate, one for each kind of plan rxi_plan_propagate makes: up to 1024 atoms one
// block per replica, split over 2 or 4 when the replicas would leave SMs idle (or RX_CLUSTER asks), per-state moves
// always unsplit; above 1024 atoms the compact layout over 2, 4 or 8 blocks, with or without per-state moves.
template <int CL_, bool PS_, bool COMPACT_> struct Layout {
    static constexpr int cl = CL_;
    static constexpr bool ps = PS_, compact = COMPACT_;
};
template <typename... L> struct LayoutList {};
using PropagateLayouts = LayoutList<
    Layout<1, false, false>, Layout<2, false, false>, Layout<4, false, false>,  // <= 1024 atoms; 2 or 4: few replicas
    Layout<1, true, false>,                                                      // <= 1024 atoms, per-state moves
    Layout<2, false, true>, Layout<4, false, true>, Layout<8, false, true>,      // > 1024 atoms
    Layout<2, true, true>, Layout<4, true, true>, Layout<8, true, true>>;        // > 1024 atoms, per-state moves

// f(Layout<...>) for the layout of the plan; false when no instantiation has it.
template <typename F, int... CL, bool... PS, bool... CP>
static bool with_layout(LayoutList<Layout<CL, PS, CP>...>, const rx_propagate_plan &plan, bool per_state, int &rc, F &&f) {
    bool found = false;
    ((!found && plan.cluster == CL && per_state == PS && (plan.compact != 0) == CP ? (found = true, rc = f(Layout<CL, PS, CP>{}))
                                                                                  : 0), ...);
    return found;
}

int rxi_propagate(rx_engine *h, uint64_t seed, uint64_t iteration, int reassign, int *launches, const int *d_only) {
    if (h->kloc == 0) return RX_OK;
    DynParams p;
    fill_dyn(h, p, reassign);
    const int N = h->cfg.n_atoms;
    if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) {
        if (!h->state_moves.empty()) RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_propagate: per-state moves are not provided for molecules");
        const uint2 mkey = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(iteration >> 32));
        const MolDev *md = (const MolDev *)h->mol_dev;
        const MolGB *gb = (const MolGB *)h->mol_gb;
        const bool no_star = getenv("RX_MOL_NO_STAR") != nullptr;   // cross-check: the general cluster path for every molecule
        const bool star = md->max_cluster <= 3 && !no_star;
        auto kern = gb ? (star ? k_propagate_mol<true, true> : k_propagate_mol<false, true>)
                       : (star ? k_propagate_mol<true, false> : k_propagate_mol<false, false>);
        const int dyn = mol_dyn_bytes(*md, gb, true);
        const int rco = smem_opt_in(h, (const void *)kern, dyn);
        if (rco) return rco;
        kern<<<h->kloc, 32 * MOL_WARPS, dyn, h->stream>>>(*md, p.move, (const StateDev *)h->d_states, (const int *)h->d_perm, (double *)h->d_pos,
                                                            (double *)h->d_vel, h->k0, mkey, (uint32_t)iteration, reassign, h->d_pot,
                                                            h->d_kin, h->d_nan, d_only, gb ? *gb : MolGB{});
        RX_CHECK_CUDA(h, cudaGetLastError());
        (*launches)++;
        return RX_OK;
    }
    const bool per_state = !h->state_moves.empty();
    if (per_state) {
        int rcm = rxi_upload_state_moves(h);
        if (rcm) return rcm;
    }
    rx_propagate_query q;
    memset(&q, 0, sizeof(q));
    q.system_kind = h->cfg.system_kind; q.n_atoms = N; q.kloc = h->kloc; q.per_state = per_state ? 1 : 0;
    q.n_sm = h->n_sm; q.smem_optin = h->smem_optin;
    for (int d = 0; d < 3; d++) q.box[d] = h->cfg.box[d];
    q.r_cutoff = h->cfg.r_cutoff;
    const char *so = getenv("RX_SKIN"), *si = getenv("RX_SKIN_IN");
    q.skin_out = so ? atof(so) : -1.0; q.skin_in = si ? atof(si) : -1.0;
    if (const char *e = getenv("RX_CLUSTER")) q.cluster = atoi(e);
    q.no_list = getenv("RX_NO_VERLET") != nullptr; q.no_sort = getenv("RX_NO_SORT") != nullptr;
    rx_propagate_plan plan;
    const int rcp = rxi_plan_propagate(&q, &plan, h->err);
    if (rcp) return rcp;
    const int cl = plan.cluster, threads = plan.threads;
    if (plan.list_capacity > 0) {
        const ListGeom g = list_geometry(&q);
        p.maxnb = plan.list_capacity;
        p.sort_atoms = plan.sort_atoms;
        p.rl2 = (float)(g.rl * g.rl);
        p.rin2 = (float)((h->cfg.r_cutoff + g.skin_in) * (h->cfg.r_cutoff + g.skin_in));
        p.half_in2 = (float)(0.25 * g.skin_in * g.skin_in);
        p.half_out2 = (float)(0.25 * (g.eff_out - g.skin_in) * (g.eff_out - g.skin_in));
    }
    const size_t smem = (size_t)plan.smem_bytes;
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(iteration >> 32));
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3((unsigned)(h->kloc * cl));
    lc.blockDim = dim3((unsigned)threads);
    lc.dynamicSmemBytes = smem;
    lc.stream = h->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    lc.attrs = at;
    lc.numAttrs = 1;
    const uint32_t it32 = (uint32_t)iteration;
    const double min_edge = 2.0 * h->cfg.r_cutoff;
    const bool npt = h->npt;
    int rc = RX_OK;
    const bool found = with_flag(p.c_is_6, [&](auto c6) {
        return with_flag(p.use_switch, [&](auto sw) {
            return with_flag(npt, [&](auto np) {
                return with_flag(h->two_regions, [&](auto rg) {
                    return with_layout(PropagateLayouts{}, plan, per_state, rc, [&](auto L) {
                        return launch_kernel(h, lc, smem > 48 * 1024, k_propagate<c6, sw, L.cl, L.ps, L.compact, np, rg>, p,
                                             (const float4 *)h->d_atom, (const StateDev *)h->d_states, (const int *)h->d_perm,
                                             h->d_pos, h->d_vel, h->k0, key, it32, h->d_pot, h->d_kin, h->d_nan, d_only,
                                             (const MoveDev *)h->d_moves, h->d_box, h->d_baro, (const double2 *)h->d_npt, min_edge);
                    });
                });
            });
        });
    });
    if (!found) RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_propagate: no kernel for the launch plan");
    if (rc) return rc;
    RX_CHECK_CUDA(h, cudaGetLastError());
    (*launches)++;
    return RX_OK;
}

// Start-of-iteration snapshot of positions and velocities (the restart policy of mcmc.py:706-759 retries a failed replica
// from the state it had when the move began) and the restore of the replicas whose NaN flag is set.
int rxi_snapshot_state(rx_engine *h) {
    if (h->kloc == 0) return RX_OK;
    const size_t bytes = (h->cfg.system_kind == RX_SYSTEM_MOLECULE ? 3 * sizeof(double) : sizeof(float4)) * (size_t)h->kloc * h->cfg.n_atoms;
    if (!h->d_pos_snap) {
        RX_CHECK_CUDA(h, cudaMalloc(&h->d_pos_snap, bytes));
        RX_CHECK_CUDA(h, cudaMalloc(&h->d_vel_snap, bytes));
        RX_CHECK_CUDA(h, cudaMalloc(&h->d_retry, sizeof(int) * h->cfg.n_replicas));
    }
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_pos_snap, h->d_pos, bytes, cudaMemcpyDeviceToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_vel_snap, h->d_vel, bytes, cudaMemcpyDeviceToDevice, h->stream));
    if (h->npt) {
        RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_box_snap, h->d_box, sizeof(double4) * h->kloc, cudaMemcpyDeviceToDevice, h->stream));
        RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_baro_snap, h->d_baro, sizeof(rx_barostat_state) * h->kloc, cudaMemcpyDeviceToDevice, h->stream));
    }
    h->have_snapshot = true;
    return RX_OK;
}

// retry[k] = the NaN flag of replica k; a failed replica's rows of positions and velocities (`words` 8-byte words each)
// and, under NPT (box != nullptr), its box and barostat state go back to the snapshot.
__global__ void k_restore_failed(const int *__restrict__ nan_flag, int *__restrict__ retry, int k0, int words,
                                 const unsigned long long *__restrict__ pos_snap, const unsigned long long *__restrict__ vel_snap,
                                 unsigned long long *__restrict__ pos, unsigned long long *__restrict__ vel,
                                 const double4 *__restrict__ box_snap, const rx_barostat_state *__restrict__ baro_snap,
                                 double4 *__restrict__ box, rx_barostat_state *__restrict__ baro) {
    const int r = blockIdx.x, k = k0 + r;
    const int failed = nan_flag[k];
    if (threadIdx.x == 0) retry[k] = failed;
    if (!failed) return;
    for (int q = threadIdx.x; q < words; q += blockDim.x) {
        pos[(size_t)r * words + q] = pos_snap[(size_t)r * words + q];
        vel[(size_t)r * words + q] = vel_snap[(size_t)r * words + q];
    }
    if (box && threadIdx.x == 0) { box[r] = box_snap[r]; baro[r] = baro_snap[r]; }
}

int rxi_restore_failed(rx_engine *h) {
    if (h->kloc == 0) return RX_OK;
    if (!h->have_snapshot) RX_FAIL(h, RX_ERR_INVALID, "rx_propagate_retry: no start-of-iteration snapshot (call rx_propagate first)");
    // a molecule's rows are double[N][3], an LJ replica's float4[N]
    const int words = (h->cfg.system_kind == RX_SYSTEM_MOLECULE ? 3 : 2) * h->cfg.n_atoms;
    using W = unsigned long long;
    k_restore_failed<<<h->kloc, 256, 0, h->stream>>>(h->d_nan, h->d_retry, h->k0, words, (const W *)h->d_pos_snap,
                                                    (const W *)h->d_vel_snap, (W *)h->d_pos, (W *)h->d_vel, h->d_box_snap,
                                                    h->d_baro_snap, h->npt ? h->d_box : nullptr, h->d_baro);
    RX_CHECK_CUDA(h, cudaGetLastError());
    return RX_OK;
}

// ---------------------------------------------------------------------------------------------------
// Energy minimisation of every owned replica in its current state: MultiStateSampler.minimize
// (multistatesampler.py:612-647) -> _minimize_replica (:1339-1402), which runs a FIRE descent first
// (integrators.py FIREMinimizationIntegrator).  FIRE as published (Bitzek et al., PRL 97, 170201 (2006)):
// semi-implicit Euler dynamics with the velocity steered towards the force, the time step grown while the power
// F.v stays positive and the motion stopped when it turns negative; plus a cap on the displacement per step so the
// overlapping starts of the reference's test systems cannot blow up.  One CTA per replica, all-pairs forces (this is a
// set-up step, not the hot path).  Velocities are left untouched.
// APT atoms per thread: thread t owns atoms t, t + nthr, ... (APT = 1 up to 1024 atoms, 4 above); its terms of the block
// sums are added in that order, so the result does not depend on scheduling.  Shared memory: [stride] positions, then
// [stride] parameter records, stride = RX_MAX_ATOMS (APT = 1) or N.
// ---------------------------------------------------------------------------------------------------
// NPT: every replica at its own box (box[r]).  REG: two alchemical regions, as in k_propagate.
template <bool C6, bool SW, int APT, bool NPT = false, bool REG = false>
__global__ void __launch_bounds__(1024) k_minimize(DynParams p, const float4 *__restrict__ atom,
                                                   const StateDev *__restrict__ states, const int *__restrict__ perm,
                                                   float4 *__restrict__ pos, int k0, float tol_rms, int max_iter,
                                                   double *__restrict__ rms_out, int *__restrict__ iters_out,
                                                   const double4 *__restrict__ box) {
    extern __shared__ float4 s_dyn[];
    BoxF bf = p.box;
    if constexpr (NPT) { const double4 b = box[blockIdx.x]; bf = box_f(b.x, b.y, b.z); }
    const int stride = APT == 1 ? RX_MAX_ATOMS : p.N;
    float4 *s_pos = s_dyn, *s_par = s_dyn + stride;
    __shared__ float s_part[32][3];
    __shared__ float s_sum[3];
    const int r = blockIdx.x, k = k0 + r, t = threadIdx.x, nthr = blockDim.x, nw = nthr >> 5;
    const StateDev st = states[perm[k]];
    float vx[APT], vy[APT], vz[APT];
#pragma unroll
    for (int u = 0; u < APT; u++) {
        const int a = t + u * nthr;
        vx[u] = vy[u] = vz[u] = 0.f;
        if (a < p.N) {
            const float4 a4 = atom[a], x4 = pos[(size_t)r * p.N + a];
            s_pos[a] = make_float4(x4.x, x4.y, x4.z, a4.x);
            s_par[a] = make_float4(a4.y, REG ? a4.w : (a4.w != 0.f ? 1.f : 0.f), 0.f, 0.f);
        }
    }
    __syncthreads();
    PairCtx pc;
    pc.box = bf; pc.rc2 = p.rc2;
    pc.lam = {(float)st.la, (float)st.ob};
    if constexpr (REG) pc.lam2 = {(float)st.la2, (float)st.ob2};

    const unsigned pos_base = (unsigned)__cvta_generic_to_shared(s_dyn);
    const float hx0 = (float)st.ho_x0[0], hx1 = (float)st.ho_x0[1], hx2 = (float)st.ho_x0[2], hK = (float)st.ho_K;
    const float dt0 = 0.001f, dt_max = 0.010f, alpha0 = 0.1f, max_move = 0.01f;  // ps, ps, -, nm per step
    float dt = dt0, alpha = alpha0;
    int n_pos = 0, it = 0;
    float rms = 0.f;
    for (;;) {
        float fx[APT], fy[APT], fz[APT], q0 = 0.f, q1 = 0.f, q2 = 0.f;
#pragma unroll
        for (int u = 0; u < APT; u++) {
            const int a = t + u * nthr;
            const bool active = a < p.N;
            const float4 xa = active ? s_pos[a] : make_float4(0, 0, 0, 0);
            float gx = 0.f, gy = 0.f, gz = 0.f, e = 0.f;
            if (p.kind == RX_SYSTEM_HARMONIC) { gx = -hK * (xa.x - hx0); gy = -hK * (xa.y - hx1); gz = -hK * (xa.z - hx2); }
            else if (active) {
                const float4 a4 = atom[a];
                pc.x = xa.x; pc.y = xa.y; pc.z = xa.z; pc.sig_i = a4.x; pc.se_i = a4.y; pc.alch_i = a4.w != 0.f;
                if constexpr (REG) pc.reg_i = (int)a4.w;
                lj_forces<C6, SW, false, false, REG>(p, pc, pos_base, 16 * stride, 0u, p.N, p.N, a, false, 0, gx, gy, gz, e);
            }
            if (!active) { gx = gy = gz = 0.f; }
            fx[u] = gx; fy[u] = gy; fz[u] = gz;
            // this thread's terms of F.F, F.v, v.v in atom order
            const float f2 = gx * gx + gy * gy + gz * gz, fv = gx * vx[u] + gy * vy[u] + gz * vz[u],
                        v2 = vx[u] * vx[u] + vy[u] * vy[u] + vz[u] * vz[u];
            if (u == 0) { q0 = f2; q1 = fv; q2 = v2; } else { q0 += f2; q1 += fv; q2 += v2; }
        }
        // block sums of F.F, F.v, v.v (fixed order: deterministic)
        for (int o = 16; o > 0; o >>= 1) {
            q0 += __shfl_down_sync(0xffffffffu, q0, o); q1 += __shfl_down_sync(0xffffffffu, q1, o); q2 += __shfl_down_sync(0xffffffffu, q2, o);
        }
        if ((t & 31) == 0) { s_part[t >> 5][0] = q0; s_part[t >> 5][1] = q1; s_part[t >> 5][2] = q2; }
        __syncthreads();  // also: every thread has finished reading the positions
        if (t < 3) { float s = 0.f; for (int w = 0; w < nw; w++) s += s_part[w][t]; s_sum[t] = s; }
        __syncthreads();
        const float FF = s_sum[0], P = s_sum[1], VV = s_sum[2];
        rms = sqrtf(FF / (3.0f * (float)p.N));
        if (!(rms > tol_rms) || it >= max_iter) break;  // converged, out of iterations, or NaN
        it++;
        const float alpha_v = alpha;
        const float mix = P > 0.f ? alpha * sqrtf(VV / fmaxf(FF, 1e-30f)) : 0.f;
        if (P > 0.f) {
            if (++n_pos > 5) { dt = fminf(dt * 1.1f, dt_max); alpha *= 0.99f; }
        } else {
            dt *= 0.5f; alpha = alpha0; n_pos = 0;
        }
#pragma unroll
        for (int u = 0; u < APT; u++) {
            const int a = t + u * nthr;
            const bool active = a < p.N;
            float wx = vx[u], wy = vy[u], wz = vz[u];
            if (P > 0.f) {
                wx = (1.f - alpha_v) * wx + mix * fx[u]; wy = (1.f - alpha_v) * wy + mix * fy[u]; wz = (1.f - alpha_v) * wz + mix * fz[u];
            } else {
                wx = wy = wz = 0.f;
            }
            const float inv_m = active ? atom[a].z : 1.f;
            wx += dt * fx[u] * inv_m; wy += dt * fy[u] * inv_m; wz += dt * fz[u] * inv_m;
            float mx = dt * wx, my = dt * wy, mz = dt * wz;
            const float m2 = mx * mx + my * my + mz * mz;
            if (m2 > max_move * max_move) {  // displacement cap: rescale this atom's velocity
                const float sc = max_move * rsqrtf(m2);
                wx *= sc; wy *= sc; wz *= sc; mx *= sc; my *= sc; mz *= sc;
            }
            vx[u] = wx; vy[u] = wy; vz[u] = wz;
            if (active) { const float4 xa = s_pos[a]; s_pos[a] = make_float4(xa.x + mx, xa.y + my, xa.z + mz, xa.w); }
        }
        __syncthreads();
    }
    if (t == 0) { rms_out[k] = (double)rms; iters_out[k] = it; }
#pragma unroll
    for (int u = 0; u < APT; u++) {
        const int a = t + u * nthr;
        if (a < p.N) {
            const float4 xa = s_pos[a];
            float x = xa.x, y = xa.y, z = xa.z;
            if (p.kind != RX_SYSTEM_HARMONIC) wrap_into(bf, x, y, z);
            pos[(size_t)r * p.N + a] = make_float4(x, y, z, 0.f);
        }
    }
}

int rxi_minimize(rx_engine *h, double tolerance, int max_iterations, double *d_rms, int *d_iters) {
    if (h->kloc == 0) return RX_OK;
    if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) {
        const MolDev *m = (const MolDev *)h->mol_dev;
        const MolGB *gb = (const MolGB *)h->mol_gb;
        auto kern = gb ? k_minimize_mol<true> : k_minimize_mol<false>;
        const int dyn = mol_dyn_bytes(*m, gb, false);
        const int rco = smem_opt_in(h, (const void *)kern, dyn);
        if (rco) return rco;
        kern<<<h->kloc, 32, dyn, h->stream>>>(*m, (double *)h->d_pos, h->k0, tolerance, max_iterations > 0 ? max_iterations : 100000,
                                              d_rms, d_iters, gb ? *gb : MolGB{});
        RX_CHECK_CUDA(h, cudaGetLastError());
        return RX_OK;
    }
    DynParams p;
    fill_dyn(h, p, 0);
    const int N = h->cfg.n_atoms;
    if (h->cfg.system_kind == RX_SYSTEM_HARMONIC && N > RX_MAX_ATOMS)
        RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_minimize: more than 1024 atoms per replica of a harmonic system is not supported");
    if (N > RX_MAX_ATOMS_LJ)
        RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_minimize: more than 4096 atoms per replica is not supported");
    // up to 1024 atoms one atom per thread; above, four per thread with 32 bytes of shared memory per atom (opted in)
    const bool wide = N > RX_MAX_ATOMS;
    const int threads = wide ? ((N + 4 * 32 - 1) / (4 * 32)) * 32 : ((N + 31) / 32) * 32;
    const size_t smem = (size_t)2 * (wide ? N : RX_MAX_ATOMS) * sizeof(float4);
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3((unsigned)h->kloc);
    lc.blockDim = dim3((unsigned)threads);
    lc.dynamicSmemBytes = smem;
    lc.stream = h->stream;
    const int rc = with_flag(p.c_is_6, [&](auto c6) {
        return with_flag(p.use_switch, [&](auto sw) {
            return with_flag(h->npt, [&](auto np) {
                return with_flag(wide, [&](auto w) {
                    return with_flag(h->two_regions, [&](auto rg) {
                        return launch_kernel(h, lc, wide, k_minimize<c6, sw, w ? 4 : 1, np, rg>, p, (const float4 *)h->d_atom,
                                             (const StateDev *)h->d_states, (const int *)h->d_perm, h->d_pos, h->k0,
                                             (float)tolerance, max_iterations, d_rms, d_iters, (const double4 *)h->d_box);
                    });
                });
            });
        });
    });
    if (rc) return rc;
    RX_CHECK_CUDA(h, cudaGetLastError());
    return RX_OK;
}

int rxi_randomize_velocities(rx_engine *h, uint64_t seed, uint64_t stream_id) {
    if (h->kloc == 0) return RX_OK;
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) {   // (k_propagate_mol projects incoming velocities onto the constraints)
        k_randomize_velocities_mol<<<h->kloc, 32, 0, h->stream>>>(*(const MolDev *)h->mol_dev, (const StateDev *)h->d_states,
                                                                 (const int *)h->d_perm, (double *)h->d_vel, h->k0, key, (uint32_t)stream_id);
        RX_CHECK_CUDA(h, cudaGetLastError());
        RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
        return RX_OK;
    }
    k_randomize_velocities<<<h->kloc, 256, 0, h->stream>>>(h->cfg.n_atoms, h->d_atom, h->d_states, h->d_perm, h->d_vel, h->k0,
                                                           key, (uint32_t)stream_id);
    RX_CHECK_CUDA(h, cudaGetLastError());
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return RX_OK;
}

// The f64 energy parameters of the engine's system (k_energy_rows, k_mc_move) for a table of n_states states.
static EnParams en_params(const rx_engine *h, int n_states) {
    const rx_config &c = h->cfg;
    EnParams p;
    memset(&p, 0, sizeof(p));
    p.N = c.n_atoms; p.M = n_states; p.kind = c.system_kind; p.n_alch = h->n_alch;
    p.Lx = c.box[0]; p.Ly = c.box[1]; p.Lz = c.box[2];
    p.rc2 = c.r_cutoff * c.r_cutoff; p.rs = c.r_switch; p.rc = c.r_cutoff;
    p.inv_w = 1.0 / (c.r_cutoff - c.r_switch);
    p.use_switch = c.use_switch; p.annihilate = h->two_regions ? h->annihilate_mask : c.annihilate_sterics;
    p.c_is_6 = (c.softcore_c == 6.0); p.sc_c = c.softcore_c;
    p.pair_cap = h->pair_cap;
    return p;
}

// Energy rows of the owned replicas at `n_states` states described by the device table `d_states`, written to
// d_out[K][n_states] (rows [k0, k0+kloc)).  The resident table/matrix are the default.
int rxi_compute_energy_rows_at(rx_engine *h, const StateDev *d_states, int n_states, double *d_out, int *launches,
                               const double2 *d_npt_tab) {
    if (h->kloc == 0) return RX_OK;
    const rx_config &c = h->cfg;
    if (c.system_kind == RX_SYSTEM_MOLECULE) {
        const MolDev *m = (const MolDev *)h->mol_dev;
        const MolGB *gb = (const MolGB *)h->mol_gb;
        auto kern = gb ? k_energy_mol<true> : k_energy_mol<false>;
        const int dyn = mol_dyn_bytes(*m, gb, false);
        const int rco = smem_opt_in(h, (const void *)kern, dyn);
        if (rco) return rco;
        kern<<<h->kloc, 32, dyn, h->stream>>>(*m, d_states, n_states, (const double *)h->d_pos, h->k0, d_out, gb ? *gb : MolGB{});
        RX_CHECK_CUDA(h, cudaGetLastError());
        (*launches)++;
        return RX_OK;
    }
    const EnParams p = en_params(h, n_states);
    const size_t smem = (size_t)3 * c.n_atoms * sizeof(double);
    if (h->npt && !d_npt_tab)
        RX_FAIL(h, RX_ERR_INVALID, "rx_compute_energies_at: a constant-pressure engine needs the states' pressures (rx_compute_energies_at_npt)");
    if (!h->npt && d_npt_tab)
        RX_FAIL(h, RX_ERR_INVALID, "rx_compute_energies_at_npt: the engine has no pressure (rx_set_pressures)");
    auto kern = h->two_regions ? (h->npt ? k_energy_rows<true, true> : k_energy_rows<false, true>)
                               : (h->npt ? k_energy_rows<true> : k_energy_rows<false>);
    const int rco = smem_opt_in(h, (const void *)kern, (int)smem);
    if (rco) return rco;
    kern<<<h->kloc, 512, smem, h->stream>>>(p, h->d_atom_d, h->d_alch_list, d_states, h->d_pos, h->k0,
                                           (double2 *)h->d_pairs, d_out, h->d_err, h->d_box, d_npt_tab);
    RX_CHECK_CUDA(h, cudaGetLastError());
    (*launches)++;
    return RX_OK;
}

int rxi_compute_energy_rows(rx_engine *h, int *launches) {
    return rxi_compute_energy_rows_at(h, h->d_states, h->cfg.n_states, h->d_u, launches, h->npt ? h->d_npt : nullptr);
}


// ---------------------------------------------------------------------------------------------------
// Molecule tables (rx_set_molecule): the term list with its slots, packed in f32 and in f64; constraint clusters.
// ---------------------------------------------------------------------------------------------------
template <typename T>
static int mol_upload(rx_engine *h, const std::vector<T> &v, const T **out) {
    void *d = nullptr;
    const size_t bytes = sizeof(T) * (v.empty() ? 1 : v.size());
    RX_CHECK_CUDA(h, cudaMalloc(&d, bytes));
    RX_CHECK_CUDA(h, cudaMemset(d, 0, bytes));
    if (!v.empty()) RX_CHECK_CUDA(h, cudaMemcpy(d, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
    h->mol_allocs.push_back(d);
    *out = (const T *)d;
    return RX_OK;
}

struct MolTermList {   // every term once with the slots of its contributions; parameters in f64
    std::vector<TBond<double>> b;
    std::vector<TAngle<double>> a;
    std::vector<TTors<double>> t;
    std::vector<TPair<double>> p;   // the plain pairs (the first n_plain), then the exceptions
    int n_plain = 0;
    std::vector<int> goff;
};

// A plain pair's epsilon: the f32 table has always held the rounded sqrt(eps_i eps_j), the f64 evaluation the product of the
// square roots; each precision keeps its expression, so that neither result changes.
static void mol_pair_eps(float &e, double ei, double ej) { e = (float)sqrt(ei * ej); }
static void mol_pair_eps(double &e, double ei, double ej) { e = sqrt(ei) * sqrt(ej); }

// The term list in precision T as one blob: MolTerms, then the four tables and goff, each padded to 16 bytes.
template <typename T>
static std::vector<unsigned char> mol_pack(const MolTermList &L, const std::vector<double> &eps) {
    std::vector<TBond<T>> b;
    std::vector<TAngle<T>> a;
    std::vector<TTors<T>> t;
    std::vector<TPair<T>> p;
    for (const auto &x : L.b) b.push_back({x.i, x.j, x.si, x.sj, (T)x.K, (T)x.r0});
    for (const auto &x : L.a) a.push_back({x.i, x.j, x.k, x.si, x.sj, x.sk, (T)x.K, (T)x.t0});
    for (const auto &x : L.t) t.push_back({x.i, x.j, x.k, x.l, x.si, x.sj, x.sk, x.sl, (T)x.n, (T)x.phase, (T)x.kk});
    for (size_t q = 0; q < L.p.size(); q++) {
        const auto &x = L.p[q];
        p.push_back({x.i, x.j, x.si, x.sj, (T)x.qq, (T)x.sig, (T)x.eps});
        if ((int)q < L.n_plain) mol_pair_eps(p.back().eps, eps[x.i], eps[x.j]);
    }
    auto up = [](size_t bytes) { return (bytes + 15) & ~(size_t)15; };
    MolTerms hd;
    memset(&hd, 0, sizeof(hd));
    size_t off = up(sizeof(MolTerms));
    hd.o_bond = (int)off; off += up(sizeof(TBond<T>) * b.size());
    hd.o_angle = (int)off; off += up(sizeof(TAngle<T>) * a.size());
    hd.o_tors = (int)off; off += up(sizeof(TTors<T>) * t.size());
    hd.o_pair = (int)off; off += up(sizeof(TPair<T>) * p.size());
    hd.o_goff = (int)off; off += up(sizeof(int) * L.goff.size());
    std::vector<unsigned char> blob(off, 0);
    memcpy(blob.data(), &hd, sizeof(hd));
    auto put = [&](int o, const auto &v) { if (!v.empty()) memcpy(blob.data() + o, v.data(), sizeof(v[0]) * v.size()); };
    put(hd.o_bond, b); put(hd.o_angle, a); put(hd.o_tors, t); put(hd.o_pair, p); put(hd.o_goff, L.goff);
    return blob;
}

// What no block of the molecule kernels (vacuum, or GB with g) can hold is refused here rather than at launch (which opts in
// above 48 KB: smem_opt_in).  The slot indices of the term tables are shorts; tables that fit in shared memory have far fewer
// slots, checked all the same.
static int mol_check_shared(rx_engine *h, const MolDev &m, const MolGB *g, const char *what) {
    int dev = 0, optin = 0;
    RX_CHECK_CUDA(h, cudaGetDevice(&dev));
    RX_CHECK_CUDA(h, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const struct { const void *kern; int dyn; } use[] = {
        {g ? (const void *)k_propagate_mol<true, true> : (const void *)k_propagate_mol<true, false>, mol_dyn_bytes(m, g, true)},
        {g ? (const void *)k_propagate_mol<false, true> : (const void *)k_propagate_mol<false, false>, mol_dyn_bytes(m, g, true)},
        {g ? (const void *)k_minimize_mol<true> : (const void *)k_minimize_mol<false>, mol_dyn_bytes(m, g, false)},
        {g ? (const void *)k_energy_mol<true> : (const void *)k_energy_mol<false>, mol_dyn_bytes(m, g, false)}};
    size_t need = 0;
    for (const auto &u : use) {
        cudaFuncAttributes fa;
        RX_CHECK_CUDA(h, cudaFuncGetAttributes(&fa, u.kern));
        need = std::max(need, fa.sharedSizeBytes + (size_t)u.dyn);
    }
    if (need > (size_t)optin || m.n_slots > 32767)
        RX_FAIL(h, RX_ERR_UNSUPPORTED, std::string(what) + " need " + std::to_string(need) +
                                           " bytes of shared memory per block, more than the device's " + std::to_string(optin));
    return RX_OK;
}

int rxi_set_molecule(rx_engine *h, const rx_molecule *mol) {
    const int n = h->cfg.n_atoms;
    if (n > MOL_MAX_ATOMS) RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_set_molecule: more than 32 atoms per molecule is not provided");
    if (!mol->mass || !mol->charge || !mol->sigma || !mol->epsilon) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: null per-atom arrays");
    auto atom_ok = [&](double v) { return v >= 0 && v < n && v == floor(v); };
    rxi_free_molecule(h);         // (a refused molecule leaves the engine without one, not with freed tables)
    h->have_particles = false;
    std::vector<double> mass(mol->mass, mol->mass + n), charge(mol->charge, mol->charge + n), sigma(mol->sigma, mol->sigma + n),
        eps(mol->epsilon, mol->epsilon + n);
    for (int i = 0; i < n; i++)
        if (!(mass[i] > 0) || !(sigma[i] > 0) || eps[i] < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: need mass > 0, sigma > 0, epsilon >= 0");
    // the term list: every term once; each atom's contributions get consecutive slots in the order bonds, angles, torsions,
    // pairs (the plain ones by partner index, then the exceptions in list order), each kind in list order
    MolTermList L;
    struct Contrib { int kind, term, role; };
    std::vector<std::vector<Contrib>> per_atom(n);
    std::vector<unsigned> nb_mask(n);   // bit j of nb_mask[i]: the pair (i, j) has the plain Coulomb + LJ interaction
    for (int i = 0; i < n; i++) nb_mask[i] = (n == 32 ? 0xffffffffu : ((1u << n) - 1u)) & ~(1u << i);
    for (int b = 0; b < mol->n_bonds; b++) {
        const double *q = mol->bonds + 4 * b;
        if (!atom_ok(q[0]) || !atom_ok(q[1]) || q[0] == q[1]) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: bad bond");
        L.b.push_back({(short)q[0], (short)q[1], 0, 0, q[2], q[3]});
        for (int r = 0; r < 2; r++) per_atom[(int)q[r]].push_back({0, b, r});
    }
    for (int a = 0; a < mol->n_angles; a++) {
        const double *q = mol->angles + 5 * a;
        if (!atom_ok(q[0]) || !atom_ok(q[1]) || !atom_ok(q[2])) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: bad angle");
        L.a.push_back({(short)q[0], (short)q[1], (short)q[2], 0, 0, 0, q[3], q[4]});
        for (int r = 0; r < 3; r++) per_atom[(int)q[r]].push_back({1, a, r});
    }
    for (int t = 0; t < mol->n_torsions; t++) {
        const double *q = mol->torsions + 7 * t;
        if (!atom_ok(q[0]) || !atom_ok(q[1]) || !atom_ok(q[2]) || !atom_ok(q[3])) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: bad torsion");
        L.t.push_back({(short)q[0], (short)q[1], (short)q[2], (short)q[3], 0, 0, 0, 0, q[4], q[5], q[6]});
        for (int r = 0; r < 4; r++) per_atom[(int)q[r]].push_back({2, t, r});
    }
    for (int e = 0; e < mol->n_exclusions; e++) {
        const int64_t i = mol->exclusions[2 * e], j = mol->exclusions[2 * e + 1];
        if (i < 0 || i >= n || j < 0 || j >= n || i == j) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: bad exclusion");
        nb_mask[i] &= ~(1u << j); nb_mask[j] &= ~(1u << i);
    }
    for (int e = 0; e < mol->n_exceptions; e++) {
        const double *q = mol->exceptions + 5 * e;
        if (!atom_ok(q[0]) || !atom_ok(q[1]) || q[0] == q[1]) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: bad exception");
        const int i = (int)q[0], j = (int)q[1];
        nb_mask[i] &= ~(1u << j); nb_mask[j] &= ~(1u << i);
    }
    auto add_pair = [&](const TPair<double> &p) {
        L.p.push_back(p);
        per_atom[p.i].push_back({3, (int)L.p.size() - 1, 0}); per_atom[p.j].push_back({3, (int)L.p.size() - 1, 1});
    };
    for (int i = 0; i < n; i++)
        for (int j = i + 1; j < n; j++)
            if ((nb_mask[i] >> j) & 1u)   // (epsilon: mol_pack)
                add_pair({(short)i, (short)j, 0, 0, MOL_ONE_4PI_EPS0 * charge[i] * charge[j], 0.5 * (sigma[i] + sigma[j]), 0.0});
    L.n_plain = (int)L.p.size();
    for (int e = 0; e < mol->n_exceptions; e++) {
        const double *q = mol->exceptions + 5 * e;
        add_pair({(short)q[0], (short)q[1], 0, 0, MOL_ONE_4PI_EPS0 * q[2], q[3], q[4]});
    }
    L.goff.assign(1, 0);
    int slot = 0;
    for (int i = 0; i < n; i++) {
        for (const Contrib &c : per_atom[i]) {
            short *dst = nullptr;
            if (c.kind == 0) dst = c.role == 0 ? &L.b[c.term].si : &L.b[c.term].sj;
            else if (c.kind == 1) dst = c.role == 0 ? &L.a[c.term].si : (c.role == 1 ? &L.a[c.term].sj : &L.a[c.term].sk);
            else if (c.kind == 2) dst = c.role == 0 ? &L.t[c.term].si : (c.role == 1 ? &L.t[c.term].sj : (c.role == 2 ? &L.t[c.term].sk : &L.t[c.term].sl));
            else dst = c.role == 0 ? &L.p[c.term].si : &L.p[c.term].sj;
            *dst = (short)slot++;
        }
        L.goff.push_back(slot);
    }
    L.goff.push_back(slot);   // (padding to an even count)
    // constraint clusters: connected components, constraints kept in list order inside a cluster
    std::vector<int> comp(n);
    for (int i = 0; i < n; i++) comp[i] = i;
    auto find = [&](int x) { while (comp[x] != x) x = comp[x] = comp[comp[x]]; return x; };
    for (int c = 0; c < mol->n_constraints; c++) {
        const double *q = mol->constraints + 3 * c;
        if (!atom_ok(q[0]) || !atom_ok(q[1]) || q[0] == q[1] || !(q[2] > 0)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: bad constraint");
        comp[find((int)q[0])] = find((int)q[1]);
    }
    std::vector<int> cluster_of(n, -1), c_off(1, 0);
    std::vector<std::vector<MolCons>> cl;
    for (int c = 0; c < mol->n_constraints; c++) {
        const double *q = mol->constraints + 3 * c;
        const int root = find((int)q[0]);
        if (cluster_of[root] < 0) { cluster_of[root] = (int)cl.size(); cl.emplace_back(); }
        cl[cluster_of[root]].push_back(MolCons{(int)q[0], (int)q[1], q[2]});
    }
    if ((int)cl.size() > 32) RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_set_molecule: more than 32 constraint clusters");
    h->mol_cluster.assign(n, -1);   // (what a Monte Carlo move's subset must hold whole, rx_set_state_mc_moves)
    for (int i = 0; i < n; i++) h->mol_cluster[i] = cluster_of[find(i)];
    std::vector<MolCons> cons;
    for (auto &c : cl) { cons.insert(cons.end(), c.begin(), c.end()); c_off.push_back((int)cons.size()); }
    MolDev *m = (MolDev *)h->mol_dev;
    if (!m) { m = new MolDev(); h->mol_dev = m; }
    memset(m, 0, sizeof(*m));
    m->n = n; m->n_clusters = (int)cl.size(); m->remove_cm = mol->remove_cm_motion ? 1 : 0;
    for (auto &c : cl) m->max_cluster = std::max(m->max_cluster, (int)c.size());
    m->tol = mol->constraint_tolerance > 0 ? mol->constraint_tolerance : 1e-8;   // integrators.py constraint_tolerance default
    const std::vector<unsigned char> t32 = mol_pack<float>(L, eps), t64 = mol_pack<double>(L, eps);
    m->bytes32 = (int)t32.size(); m->bytes64 = (int)t64.size();
    m->n_tb = (int)L.b.size(); m->n_ta = (int)L.a.size(); m->n_tt = (int)L.t.size(); m->n_tp = (int)L.p.size(); m->n_slots = slot;
    int rc = mol_check_shared(h, *m, nullptr, "rx_set_molecule: the term tables");
    if (rc) { rxi_free_molecule(h); return rc; }
    const unsigned char *d32 = nullptr, *d64 = nullptr;
    if ((rc = mol_upload(h, mass, &m->mass)) || (rc = mol_upload(h, charge, &m->charge)) || (rc = mol_upload(h, c_off, &m->c_off)) ||
        (rc = mol_upload(h, cons, &m->cons)) || (rc = mol_upload(h, t32, &d32)) || (rc = mol_upload(h, t64, &d64)))
        return rc;
    m->terms32 = (const MolTerms *)d32; m->terms64 = (const MolTerms *)d64;
    h->have_particles = true;
    return RX_OK;
}

void rxi_free_molecule(rx_engine *h) {
    for (void *d : h->mol_allocs) cudaFree(d);
    h->mol_allocs.clear();
    delete (MolDev *)h->mol_dev;
    h->mol_dev = nullptr;
    rxi_free_implicit_solvent(h);
}

void rxi_free_implicit_solvent(rx_engine *h) {
    if (h->mol_gb) cudaFree((void *)((MolGB *)h->mol_gb)->atom);
    delete (MolGB *)h->mol_gb;
    h->mol_gb = nullptr;
}

// OBC implicit solvent (rx_set_implicit_solvent): the per-atom table and the constants of MolGB.  A refused call leaves the
// engine as it was.
int rxi_set_implicit_solvent(rx_engine *h, const rx_gbsa *s) {
    const MolDev *m = (const MolDev *)h->mol_dev;
    if (!m) RX_FAIL(h, RX_ERR_INVALID, "rx_set_implicit_solvent: call rx_set_molecule first");
    const int n = m->n;
    if (!s->radius || !s->scale) RX_FAIL(h, RX_ERR_INVALID, "rx_set_implicit_solvent: null per-atom arrays");
    if (!(s->offset >= 0) || !(s->solute_dielectric > 0) || !(s->solvent_dielectric > 0) || !(s->sa_energy >= 0) ||
        !(s->probe_radius >= 0) || !isfinite(s->alpha) || !isfinite(s->beta) || !isfinite(s->gamma))
        RX_FAIL(h, RX_ERR_INVALID, "rx_set_implicit_solvent: need offset >= 0, dielectrics > 0, sa_energy >= 0, probe_radius >= 0");
    std::vector<double> tab(4 * (size_t)n);
    for (int i = 0; i < n; i++) {
        const double rho = s->radius[i], sc = s->scale[i];
        if (!(rho > 0) || !(rho > s->offset) || !(sc >= 0) || !isfinite(rho) || !isfinite(sc))
            RX_FAIL(h, RX_ERR_INVALID, "rx_set_implicit_solvent: need radius > offset, radius > 0 and scale >= 0 for every atom");
        const double rt = rho - s->offset;
        tab[4 * i] = rt; tab[4 * i + 1] = sc * rt; tab[4 * i + 2] = rho;
        tab[4 * i + 3] = 4.0 * M_PI * s->sa_energy * (rho + s->probe_radius) * (rho + s->probe_radius);
    }
    MolGB g;
    memset(&g, 0, sizeof(g));
    g.alpha = s->alpha; g.beta = s->beta; g.gamma = s->gamma;
    g.pre = -MOL_ONE_4PI_EPS0 * (1.0 / s->solute_dielectric - 1.0 / s->solvent_dielectric);
    g.on = 1;
    g.prop_bytes = (int)(sizeof(double) * (4 * (size_t)n * n + 3 * (size_t)n));
    const int rc = mol_check_shared(h, *m, &g, "rx_set_implicit_solvent: the term and solvent tables");
    if (rc) return rc;
    void *d = nullptr;
    RX_CHECK_CUDA(h, cudaMalloc(&d, sizeof(double) * tab.size()));
    const cudaError_t e = cudaMemcpy(d, tab.data(), sizeof(double) * tab.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(d); RX_CHECK_CUDA(h, e); }
    rxi_free_implicit_solvent(h);
    g.atom = (const double *)d;
    h->mol_gb = new MolGB(g);
    return RX_OK;
}

#include "rx_mc.cuh"
