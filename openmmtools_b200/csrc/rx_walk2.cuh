// rx_walk2.cuh -- second-generation swap-all walker of the filter mode (included by rx_mix.cu).  One body, two coordinate
// systems: k_mix_walk2 walks SLOTS (power-of-two K <= 256: an attempt starts on every even word), k_mix_walk2c walks
// CANDIDATE indices (any other K <= 256: the words that numba's randint accepts, rx_walk2c.cuh).
//
// Same algorithm and the same results as k_mix_walk_pow2<true> (replicaexchange.py:321-349 bit for bit); what
// changes is the length of the dependent chain of one speculation round:
//   * lane <-> record mapping is FIXED (lane = record index mod 32) and the window [h, h+32) rotates over the lanes, so a
//     lane keeps its record in registers until the record leaves the window and its next record (index + 32) is
//     prefetched a whole window ahead: no shared-memory ring access on the chain (v1: LDS ring -> LDS perm -> LDS
//     image; here: LDS perm -> LDS image).  Ballots are rotated into window order with one funnel shift;
//   * records are 16 bytes {i|j<<16, back-mask, f32 log-uniform of the attempt, hop class}; the f64 log-uniform the
//     exact path needs is recomputed from the two words of the stream (same log() as the pre-pass, same value);
//   * the commit's bookkeeping (log entry, counters, promotion of the lanes that left the window) is issued after the
//     next round's permutation loads, in their latency shadow;
//   * every lane copies its own records into a shared-memory ring with cp.async, 15 windows ahead of use (see W2_RING).
// The coordinate systems differ in the visited chain (w2_chain_slots / w2_chain_cand), in where an attempt's uniform
// lies in the stream, and in the ends of the pass.  The walkers run the bulk of a pass; the last < 600 records / < 130
// attempts are left to k_mix_walk_pow2<true> (slots, on the same records, rx_walk_exact.cuh) or k_mix_walk_serial (candidates).
#pragma once

struct SlotRec2 {        // 16 bytes, one attempt's record (per slot or per candidate index), state independent
    uint32_t ij;         // i | j << 16
    uint32_t backmask;   // bit 31-b: record s-1-b shares a replica index with record s (b = 0..30)
    uint32_t lu_next;    // float bits: log of the uniform the attempt draws (slots: the two words of slot s+1), rounded to f32
    uint32_t k;          // candidates: hop class, the attempt moves on by 2 + k candidates when it draws a uniform; slots: 0
};

// f64 log-uniform of slot s
__device__ __forceinline__ double slot_logU(const uint32_t *__restrict__ words, unsigned s) {
    const double U = mt_double(words[2 * (size_t)s], words[2 * (size_t)s + 1]);
    return (U == 0.0) ? LOGU_ZERO : log(U);
}

// Slot records, state independent: the replica indices of slot s, its back-mask over the 31 slots before it, and (SlotRec) the
// f64 log-uniform of the slot itself or (SlotRec2) the f32 log-uniform of the next slot, the draw of an attempt at s.
template <bool REC2>
__global__ void __launch_bounds__(256) k_slots_build(const uint32_t *__restrict__ words, long long nslots, uint32_t mask,
                                                     std::conditional_t<REC2, SlotRec2, SlotRec> *__restrict__ rec) {
    __shared__ uint32_t s_ij[256 + 31];
    const long long s0 = (long long)blockIdx.x * 256;
    const int t = threadIdx.x;
    for (int q = t; q < 256 + 31; q += 256) {   // tile: slots s0-31 .. s0+255
        const long long s = s0 - 31 + q;
        uint32_t ij = 0xffffffffu;
        if (s >= 0 && s < nslots) ij = (words[2 * s] & mask) | ((words[2 * s + 1] & mask) << 16);
        s_ij[q] = ij;
    }
    __syncthreads();
    const long long s = s0 + t;
    if (s >= nslots) return;
    const uint32_t ij = s_ij[t + 31];
    const uint32_t i = ij & 0xffffu, j = ij >> 16;
    uint32_t bm = 0;
#pragma unroll 4
    for (int b = 0; b < 31; b++) {
        const uint32_t o = s_ij[t + 30 - b];
        const uint32_t oi = o & 0xffffu, oj = o >> 16;
        const bool hit = (o != 0xffffffffu) && (oi == i || oi == j || oj == i || oj == j);
        bm |= (hit ? 1u : 0u) << (31 - b);
    }
    if constexpr (REC2) {
        SlotRec2 r;
        r.ij = ij;
        r.backmask = bm;
        float lu = 0.f;
        if (s + 1 < nslots) lu = (float)slot_logU(words, (unsigned)(s + 1));
        r.lu_next = __float_as_uint(lu);
        r.k = 0;
        rec[s] = r;
    } else {
        SlotRec r;
        r.ij = ij;
        r.backmask = bm;
        r.logU = slot_logU(words, (unsigned)s);
        rec[s] = r;
    }
}

// The filter's decision for one (i, j, si, sj): image values d_x = image of u[x, s_x] - rowmin_x (the maintained diagonal)
// and f_xy = image of u[x, s_y] - rowmin_x.  Same rigorous bound as k_mix_walk_pow2<true> (see its derivation there;
// the factor 3.2e-5 leaves 5 % over the 2^-15 + 2^-23 the roundings need, far more than the re-association below costs):
//   e0  = 3.2e-5 (|d_i| + |d_j|) + eps0        as soon as the states are known (before the image loads return),
//   eps = 3.2e-5 (|f_ij| + |f_ji|) + e0,       lp = (d_i - f_ij) + (d_j - f_ji),
//   log_p >= 0 is certain iff lp > eps; it is certainly < 0 iff lp < -eps; the comparison with the uniform is certain
//   iff |lp - lu| > mar = 1.3e-7 (|lp| + |lu|) + eps.
// eps0 = rowabs[i] + rowabs[j] + 1e-9, or -1e30 for a slot with i == j: the reference's log_p is then exactly 0 for finite
// energies (accepted without a draw) and lp is exactly 0 > eps; non-finite energies give lp = NaN (undecided: exact path).
__device__ __forceinline__ void w2_filter(float d_i, float f_ij, float d_j, float f_ji, float e0, float lu,
                                          bool &ge0, bool &acc, bool &undecided) {
    const float lp = (d_i - f_ij) + (d_j - f_ji);
    const float eps = fmaf(fabsf(f_ij) + fabsf(f_ji), 3.2e-5f, e0);
    ge0 = lp > eps;
    const float d = lp - lu;
    const float mar = fmaf(fabsf(lp) + fabsf(lu), 1.3e-7f, eps);
    const bool dec_lp = fabsf(lp) > eps;
    acc = ge0 || (dec_lp && d > mar);
    undecided = !(ge0 || (dec_lp && fabsf(d) > mar));
}

// One entry per replica k: the walker's view of the permutation.  `diag` is the image value of u[k, state] - rowmin_k, so
// a round reads the two diagonal terms of log_p together with the states (one dependent shared-memory level less) and
// only the two off-diagonal image values afterwards.  8 bytes: two wavefronts per warp-wide access at best.
struct __align__(8) W2Replica {
    int state;
    float diag;
};

// Shared-memory accesses of the round loop by explicit 32-bit shared addresses.  (With generic pointers the compiler
// re-derives the shared window base from SR_CgaCtaId inside the loop -- an S2UR of a few hundred cycles on the chain.)
__device__ __forceinline__ uint2 w2_lds64(unsigned a) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint4 w2_lds128(unsigned a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void w2_sts64(unsigned a, unsigned x, unsigned y) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ float w2_image_at(unsigned a_hi, unsigned a_lo) {   // the image is read-only while the walker runs
    unsigned hi, lo;
    asm("ld.shared.u16 %0, [%1];" : "=r"(hi) : "r"(a_hi));
    asm("ld.shared.u8 %0, [%1];" : "=r"(lo) : "r"(a_lo));
    return __uint_as_float(__byte_perm(hi, lo, 0x1045));
}

// The walker's record ring: 16 entries per lane (= per record class mod 32), filled by the lane itself with asynchronous
// global->shared copies 15 windows ahead of use (no register, no scoreboard wait; DRAM latency is far below that);
// completion is tracked by the hardware (cp.async.wait_group): no flags, no fences, no second warp in the loop.
// (A producer warp that prepared ready-to-use contexts was tried: 106 instead of 125 instructions per round for the
// walker, but its shared-memory traffic and the acquire/release pairs made the walker's own loads wait twice as long,
// so its rounds were slower than this organisation's.)
#define W2_RING 512
__device__ __forceinline__ void w2_cp_async16(unsigned dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void w2_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void w2_cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// The exact decision for one attempt of a SlotRec2 record (ij = i | j << 16) under the states (si, sj): bit 0 = log_p >= 0,
// bit 1 = accepted.  `a` is the word position of the uniform the attempt draws if log_p < 0.  f64 energies from L2, the
// reference's own arithmetic; the uniform is compared in the log domain outside a 1e-9 band and as U < exp(log_p) inside it.
__device__ __noinline__ unsigned w2_exact_decision(const double *__restrict__ u, int K, unsigned ij, unsigned si, unsigned sj,
                                                   const uint32_t *__restrict__ words, size_t a) {
    const size_t rowi = (size_t)(ij & 0xffffu) * K, rowj = (size_t)(ij >> 16) * K;
    const double logp = swap_logp(u[rowi + sj], u[rowj + si], u[rowi + si], u[rowj + sj]);
    if (logp >= 0.0) return 3u;
    const double U = mt_double(words[a], words[a + 1]);
    const double dd = logp - ((U == 0.0) ? LOGU_ZERO : log(U));
    bool acc;
    if (dd > 1e-9) acc = true;
    else if (dd < -1e-9) acc = false;
    else acc = U < rx_exp_cr(logp);
    return acc ? 2u : 0u;
}

// Visited chain of one window of slots (window-order masks): from a visited slot the next attempt starts 1 slot later if
// log_p >= 0, else 2.  skip[s+1] = NG[s] & ~skip[s] (see k_mix_walk_pow2).  V: visited positions; Cf: visited positions at
// which the next round has to start -- position 31 when it draws a uniform: that uniform's slot lies beyond the window, and
// committing it here would make the window advance by 33 (the lane of the skipped slot would have to move on by two
// windows at once); the attempt simply opens the next round instead.
__device__ __forceinline__ void w2_chain_slots(unsigned Gw, unsigned &V, unsigned &Cf) {
    const unsigned X = ~Gw;
    const unsigned starts = X & ~(X << 1);
    const unsigned SE = starts & 0x55555555u, SO = starts & 0xAAAAAAAAu;
    const unsigned sumE = X + SE, sumO = X + SO;
    const unsigned skip = (((sumE ^ X) & ~SE) & 0xAAAAAAAAu) | (((sumO ^ X) & ~SO) & 0x55555555u);
    V = ~skip;
    Cf = X & 0x80000000u;
}

// Visited chain of one window of candidate indices: hops {2, 3, 4}.  With T = positions that would hop 3 (log_p < 0, k = 1)
// and F = positions that would hop 4 (log_p < 0, k = 2): on ONE parity class ("grid") of positions the chain is the slot
// chain (hop 2 = next grid position, hop 4 = skip one), solved for all positions at once by the add-carry trick on stride-2
// masks (the bit between two grid positions of an F-run is filled so that the carry runs through).  A visited T switches
// to the other grid; there the steady-state pattern holds from the entry position on unless the steady state skips the
// entry position, in which case the pattern of the F-run that contains it is complemented.  One grid phase per visited T
// (a uniform loop: all masks are warp-wide values).  V: visited positions, valid below and at the lowest bit of the
// returned forced stops Cf (visited positions at which the next round has to start).  tests/test_walk_cand_logic_model.py
// is the lane-level CPU model of this logic.
__device__ __forceinline__ void w2_chain_cand(unsigned Gw, unsigned K1w, unsigned K2w, unsigned &V, unsigned &Cf) {
    const unsigned NG = ~Gw;
    const unsigned T = NG & K1w, F = NG & K2w;
    // steady state of both grids (every F-run assumed to start visited)
    const unsigned XgE = F & 0x55555555u, XgO = F & 0xAAAAAAAAu;
    const unsigned XpE = XgE | (XgE << 1), XpO = XgO | (XgO << 1);
    const unsigned stE = XgE & ~(XgE << 2), stO = XgO & ~(XgO << 2);
    const unsigned sEa = XpE + (stE & 0x11111111u), sEb = XpE + (stE & 0x44444444u);
    const unsigned sOa = XpO + (stO & 0x22222222u), sOb = XpO + (stO & 0x88888888u);
    const unsigned VE = 0x55555555u & ~(((sEa ^ XpE) & 0x44444444u) | ((sEb ^ XpE) & 0x11111111u));
    const unsigned VO = 0xAAAAAAAAu & ~(((sOa ^ XpO) & 0x88888888u) | ((sOb ^ XpO) & 0x22222222u));
    // one grid phase per visited T: from position s on the current grid up to its first visited T; the F-run that contains
    // s is complemented if the steady state skips s (never the case for position 0: bit 0 of VE is set)
    unsigned Vc = VE, Xc = XpE, gc = 0x55555555u, Vn = VO, Xn = XpO, gn = 0xAAAAAAAAu;
    unsigned s = 1u;
    V = 0u;
    for (;;) {
        const unsigned R = ((Xc + s) ^ Xc) & gc;
        const unsigned Vg = (Vc ^ ((s & ~Vc) ? R : 0u)) & ~(s - 1u);
        const unsigned Tv = Vg & T, t = Tv & (0u - Tv);
        V |= Vg & ((t << 1) - 1u);          // t == 0 -> all
        s = t << 3;                          // entry of the other grid (0: no further switch inside the window)
        if (s == 0u) break;
        unsigned x;
        x = Vc; Vc = Vn; Vn = x;
        x = Xc; Xc = Xn; Xn = x;
        x = gc; gc = gn; gn = x;
    }
    // The next round has to start inside the window or right behind it (a lane moves on by one window per round at most): a
    // visited position p ends the round if p + hop(p) > 32 -- position 31 always, 30 unless it hops 2, 29 if it hops 4.  The
    // chain's last visited position either is such a position or hops to 32 exactly (then the whole window commits).
    Cf = V & (0x80000000u | ((T | F) & 0x40000000u) | (F & 0x20000000u));
}

// The walker.  CAND = false: records are slots [ctl->head, nrec); CAND = true: records are candidate indices [0, nrec), cpos
// gives the word position of every candidate.  The image is re-laid out row by row in shared memory -- u16 plane of the row
// (2K bytes), then its u8 plane (K bytes), padded to an even length -- so that one address per row serves both planes.
#define W2_THREADS 128   // warps 1.. only help with the prologue
template <bool CAND>
__device__ __forceinline__ void w2_walk(const SlotRec2 *__restrict__ rec, const uint32_t *__restrict__ words,
                                        const uint32_t *__restrict__ cpos, unsigned nrec, const double *__restrict__ u, int K,
                                        int logK, int *__restrict__ perm_g, uint32_t *__restrict__ slot_log,
                                        const unsigned char *__restrict__ filt, const double *__restrict__ filt_rowabs,
                                        MixCtl *ctl) {
    extern __shared__ uint4 s_w2[];
    __shared__ unsigned long long s_ptrs[2];               // global base pointers of the round loop (see there)
    uint4 *s_ring = s_w2;                                  // [W2_RING] records
    W2Replica *s_rep = (W2Replica *)(s_ring + W2_RING);    // [K]
    unsigned char *s_q = (unsigned char *)(s_rep + K);     // image rows
    const unsigned row_bytes = (3u * (unsigned)K + 1u) & ~1u, lo_off = 2u * (unsigned)K;
    // (the warp index through a shuffle: the compiler then knows that it is the same in all lanes, and neither guards the
    // walker's ballots against divergence nor builds its loop with divergence-capable -- slowly resolved -- branches)
    const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    {
        const unsigned short *ghi = (const unsigned short *)filt;
        const unsigned char *glo = filt + 2 * (size_t)K * K;
        if (!CAND && K >= 16) {   // 16-byte pieces: 8 values of the u16 plane, 16 of the u8 plane, never across a row
            const uint4 *ghi4 = (const uint4 *)ghi, *glo4 = (const uint4 *)glo;   // (cudaMalloc alignment, 2 K^2 % 16 == 0)
            for (int q = tid; q < (K * K) / 8; q += W2_THREADS) {
                const int e = q * 8, row = e >> logK, col = e & (K - 1);
                *(uint4 *)(s_q + (size_t)row_bytes * row + 2 * col) = ghi4[q];
            }
            for (int q = tid; q < (K * K) / 16; q += W2_THREADS) {
                const int e = q * 16, row = e >> logK, col = e & (K - 1);
                *(uint4 *)(s_q + (size_t)row_bytes * row + lo_off + col) = glo4[q];
            }
        } else {
            for (int row = warp; row < K; row += W2_THREADS / 32) {
                unsigned char *rowp = s_q + (size_t)row_bytes * row;
                for (int col = lane; col < K; col += 32) {
                    ((unsigned short *)rowp)[col] = ghi[(size_t)row * K + col];
                    rowp[lo_off + col] = glo[(size_t)row * K + col];
                }
            }
        }
    }
    if (tid == 0) { s_ptrs[0] = (unsigned long long)__cvta_generic_to_global(slot_log); s_ptrs[1] = (unsigned long long)rec; }
    __syncthreads();
    float rowabs_max = 0.f;
    for (int q = tid; q < K; q += W2_THREADS) {
        W2Replica e;
        e.state = perm_g[q];
        const unsigned char *rowp = s_q + (size_t)row_bytes * q;
        e.diag = __uint_as_float(__byte_perm((unsigned)((const unsigned short *)rowp)[e.state], (unsigned)rowp[lo_off + e.state], 0x1045));
        s_rep[q] = e;
    }
    // the rows' share of the filter's rounding bound, the largest of all rows (rounded up; K values, read by every warp)
    for (int q = lane; q < K; q += 32)
        rowabs_max = fmaxf(rowabs_max, __fmul_ru(1.6e-14f, __fadd_ru(__double2float_ru(fabs(filt_rowabs[q])), 0.5f)));
    for (int o = 16; o; o >>= 1) rowabs_max = fmaxf(rowabs_max, __shfl_xor_sync(0xffffffffu, rowabs_max, o));
    const float eps_rows = __fadd_ru(__fadd_ru(rowabs_max, rowabs_max), 1e-9f);
    __syncthreads();
    if (warp != 0) return;
    const uint4 *__restrict__ recs = (const uint4 *)rec;

    // slots: the pass continues at slot ctl->head; candidates: a pass starts at candidate 0 (word position ctl->head == 0)
    const long long head0 = ctl->head;
    unsigned h = CAND ? 0u : (unsigned)head0;
    const long long remaining0 = ctl->remaining;
    unsigned rem = remaining0 > 0x7fffffffLL ? 0x7fffffffu : (unsigned)remaining0;
    const unsigned rem0 = rem;
    unsigned rounds = 0, slow = 0;
    // a round may start while h + 99 <= h_end: its lanes copy the records up to h + 31 + 32 + 480 into the ring
    const unsigned h_end = nrec >= 1200u ? nrec - 560u : 0u;
    if ((!CAND || head0 == 0) && rem >= 130 && nrec >= 1200u && h + 99u <= h_end) {
        // 32-bit shared addresses (through a shuffle, so that they live in registers instead of being re-derived)
        const unsigned ring_base = __shfl_sync(0xffffffffu, (unsigned)__cvta_generic_to_shared((const void *)s_ring), 0);
        const unsigned rep_base = __shfl_sync(0xffffffffu, (unsigned)__cvta_generic_to_shared((const void *)s_rep), 0);
        const unsigned img_base = __shfl_sync(0xffffffffu, (unsigned)__cvta_generic_to_shared((const void *)s_q), 0);
        unsigned r = h & 31u;                           // lane of window position 0
        unsigned w = ((unsigned)lane - h) & 31u;        // this lane's window position
        unsigned sA = h + w;                            // this lane's record
        // (the two global base pointers of the loop as opaque register values: taken from the constant bank where they are
        // used, each use would wait for an LDC)
        // (read back from shared memory by a volatile load: nothing the compiler can re-derive)
        const uint2 pl = w2_lds64((unsigned)__cvta_generic_to_shared((const void *)&s_ptrs[0]));
        const uint2 pr = w2_lds64((unsigned)__cvta_generic_to_shared((const void *)&s_ptrs[1]));
        const unsigned long long slot_log_r = ((unsigned long long)pl.y << 32) | pl.x;
        const uint4 *recs_r = (const uint4 *)(((unsigned long long)pr.y << 32) | pr.x);
        // record contexts: A = the lane's record, B = its next record, one window later (its raw record is loaded a round
        // ahead): back-mask, f32 log-uniform, the filter bound's constant term (-1e30 when i == j), all-ones if i != j,
        // shared addresses of the image rows and of the replica entries of i and j, hop class (candidates)
        unsigned bmA, neqA, rowiA, rowjA, repiA, repjA, kA;
        float luA, epsA;
        // of the next record only what the commit needs at once is prepared a round ahead: its indices and the addresses
        // of its replica entries; the rest of its context is derived when (and only in the lanes where) it is entered
        unsigned iB, jB, repiB, repjB;
        auto ahead = [&](const uint4 q) {
            iB = q.x & 0xffffu; jB = q.x >> 16;
            repiB = rep_base + (iB << 3); repjB = rep_base + (jB << 3);
        };
        // ring entry of record s: s mod W2_RING; this lane owns the entries of its class (s mod 32)
        for (unsigned k = 0; k < 16u; k++) w2_cp_async16(ring_base + (((sA + 32u * k) & (W2_RING - 1)) << 4), recs + (sA + 32u * k));
        w2_cp_async_commit();
        w2_cp_async_wait<0>();
        __syncwarp();
        {
            const uint4 q = w2_lds128(ring_base + ((sA & (W2_RING - 1)) << 4));
            const unsigned i = q.x & 0xffffu, j = q.x >> 16;
            bmA = q.y; luA = __uint_as_float(q.z);
            if constexpr (CAND) kA = q.w;
            neqA = i != j ? 0xffffffffu : 0u;
            epsA = i != j ? eps_rows : -1e30f;
            rowiA = img_base + i * row_bytes; rowjA = img_base + j * row_bytes;
            repiA = rep_base + (i << 3); repjA = rep_base + (j << 3);
        }
        unsigned ridxB = (sA + 32u) & (W2_RING - 1);   // ring entry of the next record
        uint4 qB = w2_lds128(ring_base + (ridxB << 4));
        ahead(qB);
        uint2 ei = w2_lds64(repiA), ej = w2_lds64(repjA);   // {state, diag} of both replicas
        // what the round resolved last leaves to the next block: the stops (window order; the positions below the lowest one
        // leave the window, 0: all of them), the visited positions, all-ones if this lane's position is visited / is visited
        // and its attempt changes the permutation, its log entry
        unsigned p_stop = 1, p_vis = 0, p_mv = 0, p_sw = 0, p_entry = 0;
        unsigned lem = (2u << w) - 1u;   // the lane's prefix mask: window positions 0 .. w (w = 31: all)
        float f_ij = 0.f, f_ji = 0.f;
        unsigned K1w = 0, K2w = 0;   // candidates: window-order masks of the positions with k == 1 / k == 2 (state independent)
        // Commit the round described by the p_* values, slide the window and fetch the states of the next round:
        // permutation stores, at once the next round's loads, then the lane state.
        auto commit = [&]() {
            // A lane's record leaves the window iff no stop lies at or before its position: one test of the stops against
            // the lane's own prefix mask, so that the predicates of the stores are one test away from the stop mask.  The
            // committed prefix itself (`below`) is only needed for the counts, off that chain; the
            // window advances by its population count (computed here rather than at the end of the previous block: a
            // population count is a long-latency operation whose scoreboard slot would otherwise be waited for at the
            // loop's back edge).
            const bool p_promoted = (p_stop & lem) == 0u;
            const bool p_mine = p_promoted && p_mv != 0u;
            const bool p_swaps = p_promoted && p_sw != 0u;
            const unsigned p_below = (p_stop & (0u - p_stop)) - 1u;
            const unsigned p_advance = (unsigned)__popc(p_below);
            if (p_swaps) {   // replica i takes state sj: its new diagonal value is the off-diagonal one just read
                w2_sts64(repiA, ej.x, __float_as_uint(f_ij));
                w2_sts64(repjA, ei.x, __float_as_uint(f_ji));
            }
            __syncwarp();
            // the states of the next round: of the next record for the lanes that leave the window
            const uint2 ein = w2_lds64(p_promoted ? repiB : repiA), ejn = w2_lds64(p_promoted ? repjB : repjA);
            if (p_mine)   // sparse commit log, indexed by record (zero = no attempt)
                asm volatile("st.global.u32 [%0], %1;" ::"l"(slot_log_r + 4ull * sA), "r"(p_entry) : "memory");
            if (p_promoted) {
                bmA = qB.y; luA = __uint_as_float(qB.z);
                if constexpr (CAND) kA = qB.w;
                neqA = iB != jB ? 0xffffffffu : 0u;
                epsA = iB != jB ? eps_rows : -1e30f;
                rowiA = img_base + iB * row_bytes; rowjA = img_base + jB * row_bytes;
                repiA = repiB; repjA = repjB;
                sA += 32u;
                w2_cp_async16(ring_base + (((ridxB - 32u) & (W2_RING - 1)) << 4), recs_r + (sA + 480u));   // over the entry of the record just left
                ridxB = (ridxB + 32u) & (W2_RING - 1);
            }
            w2_cp_async_commit();
            // the record of the (possibly new) next record: the lanes that stay re-read the one they hold
            qB = w2_lds128(ring_base + (ridxB << 4));
            h += p_advance;
            r = (r + p_advance) & 31u;
            rem -= __popc(p_vis & p_below);
            ei = ein;
            ej = ejn;
            w = (w - p_advance) & 31u;
            lem = (2u << w) - 1u;
            if constexpr (CAND) {   // the hop classes of the new window (off the chain: they only depend on the promotions)
                const unsigned b1 = __ballot_sync(0xffffffffu, kA == 1u), b2 = __ballot_sync(0xffffffffu, kA == 2u);
                K1w = __funnelshift_r(b1, b1, r); K2w = __funnelshift_r(b2, b2, r);
            }
        };
        // the exact decision for this lane's attempt (bits as w2_exact_decision)
        auto exact = [&](unsigned si, unsigned sj) {
            const size_t a = CAND ? (size_t)cpos[sA + 1] + 1 : 2 * (size_t)(sA + 1);   // the uniform's words: a, a + 1
            return w2_exact_decision(u, K, rec[sA].ij, si, sj, words, a);
        };
        unsigned Cw = 0;
        // The fast loop ends when nothing can commit, i.e. when window position 0 is itself a stop: bit 0 of Cw.  Position 0 is
        // always visited, is never a forced stop and has no earlier position, so that bit is the `undecided` answer of the
        // lane at position 0.  Slots take it from a vote straight into a predicate: read off Cw it goes from the uniform
        // datapath's predicate to the branch (a 13-cycle fixed stall at the back edge of every round; 7 % of the round at
        // K = 256, DESIGN.md 4.1).  Candidates keep the test on Cw: their longer chain resolver hides that stall, and the
        // extra vote made their round 2.7 % slower.
        bool stop0 = false;
        // Exact decisions injected into ONE fast round (see the rare path below): `bias` joins the lane's log_p, `luA` is
        // replaced, so that the filter reproduces the exact answer; both are restored when that round has been resolved.
        float bias = 0.f, lu_saved = 0.f;
        bool injected = false;
        for (;;) {
            // ---------------- the budget and the end of the pass, every 64 rounds at most: a round commits at most 32
            // attempts and advances at most 32 records (the round resolved last stays pending across this step)
            if (rem < 130u || h + 99u > h_end) break;
            unsigned quota = min(min((rem - 97u) >> 5, (h_end - h - 66u) >> 5), injected ? 1u : 64u);
            // ---------------- fast rounds.  The loop is rotated: an iteration COMMITS the round resolved by the previous
            // one and then evaluates and resolves the next, so that the block begins with the dependent chain (stores ->
            // state loads -> image loads -> filter -> ballots); no data-dependent branch besides the loop's.
            do {
                commit();
                rounds++;
                const unsigned si = ei.x, sj = ej.x;
                f_ij = w2_image_at(rowiA + 2u * sj, rowiA + lo_off + sj);
                f_ji = w2_image_at(rowjA + 2u * si, rowjA + lo_off + si);
                const float e0 = fmaf(fabsf(__uint_as_float(ei.y)) + fabsf(__uint_as_float(ej.y)), 3.2e-5f, epsA);
                w2_cp_async_wait<8>();   // a copy is used 15 of the lane's promotions (at least 15 rounds) after it was issued
                ahead(qB);
                bool ge0, acc, undecided;
                w2_filter(__uint_as_float(ei.y), f_ij, __uint_as_float(ej.y) + bias, f_ji, e0, luA, ge0, acc, undecided);
                const unsigned und = undecided ? 1u : 0u;
                const bool changes = acc && neqA != 0u;
                const unsigned G = __ballot_sync(0xffffffffu, ge0);
                const unsigned A = __ballot_sync(0xffffffffu, changes);
                const unsigned Gw = __funnelshift_r(G, G, r), Aw = __funnelshift_r(A, A, r);   // window order
                unsigned V, Cf;
                if constexpr (CAND) w2_chain_cand(Gw, K1w, K2w, V, Cf);
                else w2_chain_slots(Gw, V, Cf);
                const unsigned VA = V & Aw;
                unsigned earlier;   // bit 31-b: window position w-1-b is a visited state-changing swap
                asm("shl.b32 %0, %1, %2;" : "=r"(earlier) : "r"(VA), "r"(32u - w));
                // A round ends before the first visited lane that is stale -- or that the filter could not decide -- and
                // at the forced stops of the chain.
                const unsigned C = __ballot_sync(0xffffffffu, ((earlier & bmA) | und) != 0u);
                Cw = (__funnelshift_r(C, C, r) | Cf) & V;   // empty: the whole window commits
                if constexpr (CAND) stop0 = (Cw & 1u) != 0u;
                else stop0 = __any_sync(0xffffffffu, undecided && w == 0u);
                p_stop = Cw; p_vis = V;
                p_mv = ((V >> w) & 1u) != 0u ? 0xffffffffu : 0u;
                p_sw = changes ? p_mv : 0u;
                p_entry = (sj * (1u << LOG_STATE_BITS) + si) | (acc ? (1u << 31) | (1u << LOG_ACC_BIT) : (1u << 31));
                // (position 0 is always visited: nothing commits iff it is itself the lane that ends the round)
            } while (--quota != 0u && !stop0);
            // (a no-op unless the round just resolved ran alone, with injected decisions: see below)
            const bool was_injected = injected;
            luA = was_injected ? lu_saved : luA;
            bias = 0.f;
            injected = false;
            if (!stop0) continue;
            commit();   // (nothing to commit: positions the lanes on the round that could not start)
            w2_cp_async_wait<8>();
            ahead(qB);
            // ---------------- rare: the filter could not decide the window's first lane (nothing was committed: the states
            // are those the round was evaluated with).  Every undecided lane takes the exact decision for its record and
            // injects it into the next fast round -- a bias of +-1e20..1e30 on its log_p and a matching log-uniform make
            // the filter reproduce it -- which is run alone (quota 1) and then resolves and commits like any other round.
            // (One exact attempt per rare event would cost 0.4 us per attempt on a degenerate matrix: at iteration 0 all
            // replicas are in the same configuration and every log_p is a rounding error around 0.)
            if (!was_injected) {
                const unsigned si = ei.x, sj = ej.x;
                const float f1 = w2_image_at(rowiA + 2u * sj, rowiA + lo_off + sj);
                const float f2 = w2_image_at(rowjA + 2u * si, rowjA + lo_off + si);
                const float e0 = fmaf(fabsf(__uint_as_float(ei.y)) + fabsf(__uint_as_float(ej.y)), 3.2e-5f, epsA);
                bool ge0, acc, undecided;
                w2_filter(__uint_as_float(ei.y), f1, __uint_as_float(ej.y), f2, e0, luA, ge0, acc, undecided);
                lu_saved = luA;
                if (undecided) {
                    const unsigned d = exact(si, sj);
                    bias = (d & 1u) ? 1e30f : -1e20f;
                    if (!(d & 1u)) luA = (d & 2u) ? -1e30f : 0.f;
                    slow++;
                }
                __syncwarp();
                injected = true;
                continue;
            }
            // ---------------- rarer still: undecided WITH the exact decision injected (non-finite energies make log_p a NaN
            // whatever the bias): one exact attempt, exactly what the reference does (window position 0 commits; positions
            // 0 .. advance-1 leave the window, as many as the attempt's hop)
            {
                rounds++;
                unsigned d = 0;
                const unsigned si = ei.x, sj = ej.x;
                f_ij = w2_image_at(rowiA + 2u * sj, rowiA + lo_off + sj);
                f_ji = w2_image_at(rowjA + 2u * si, rowjA + lo_off + si);
                if (w == 0u) { d = exact(si, sj); slow++; }
                __syncwarp();
                const bool first_ge0 = __ballot_sync(0xffffffffu, (d & 1u) != 0u) != 0u;
                const bool acc = (d & 2u) != 0u;
                p_vis = 1u;
                if constexpr (CAND) {
                    const unsigned k0 = (K1w & 1u) + 2u * (K2w & 1u);   // hop class of window position 0
                    p_stop = first_ge0 ? 4u : 4u << k0;                 // 2 or 2 + k positions leave the window
                } else {
                    p_stop = first_ge0 ? 2u : 4u;                       // 1 or 2
                }
                p_mv = w == 0u ? 0xffffffffu : 0u;
                p_sw = (acc && neqA != 0u) ? p_mv : 0u;
                p_entry = (sj * (1u << LOG_STATE_BITS) + si) | (acc ? (1u << 31) | (1u << LOG_ACC_BIT) : (1u << 31));
                commit();
                w2_cp_async_wait<8>();
                ahead(qB);
                p_stop = 1u; p_vis = 0u;
            }
        }
        commit();   // the round resolved last, if one is pending
        w2_cp_async_wait<0>();
        __syncwarp();
        for (int q = lane; q < K; q += 32) perm_g[q] = s_rep[q].state;
    }
    slow = __reduce_add_sync(0xffffffffu, slow);
    if (lane == 0) {
        const long long remaining = remaining0 - (long long)(rem0 - rem);
        if constexpr (!CAND) ctl->head = h;
        else if (h > 0) ctl->head = (long long)cpos[h];   // word position: the first word the next attempt can use as an index
        ctl->aux = h;                                      // records walked: the extent of the sparse commit log
        ctl->remaining = remaining;
        ctl->status = remaining > 0 ? 1 : 0;
        ctl->rounds += (int)rounds;
        ctl->slow_exp += slow;
    }
}

__global__ void __launch_bounds__(W2_THREADS) k_mix_walk2(const SlotRec2 *__restrict__ rec, const uint32_t *__restrict__ words,
                                                  unsigned nslots, const double *__restrict__ u, int K, int logK,
                                                  int *__restrict__ perm_g, uint32_t *__restrict__ slot_log,
                                                  const unsigned char *__restrict__ filt,
                                                  const double *__restrict__ filt_rowabs, MixCtl *ctl) {
    w2_walk<false>(rec, words, nullptr, nslots, u, K, logK, perm_g, slot_log, filt, filt_rowabs, ctl);
}

__global__ void __launch_bounds__(W2_THREADS) k_mix_walk2c(const SlotRec2 *__restrict__ rec, const uint32_t *__restrict__ words,
                                                   const uint32_t *__restrict__ cpos, const uint32_t *__restrict__ ncand_p,
                                                   const double *__restrict__ u, int K, int *__restrict__ perm_g,
                                                   uint32_t *__restrict__ slot_log, const unsigned char *__restrict__ filt,
                                                   const double *__restrict__ filt_rowabs, MixCtl *ctl) {
    const unsigned ncand = *ncand_p;   // records exist for c < ncand - 3
    w2_walk<true>(rec, words, cpos, ncand >= 3u ? ncand - 3u : 0u, u, K, 0, perm_g, slot_log, filt, filt_rowabs, ctl);
}
