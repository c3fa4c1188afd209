// rx_walk_exact.cuh -- the exact speculative swap-all walker (included by rx_mix.cu after rx_walk2.cuh).  One body, two
// coordinate systems: k_mix_walk_pow2 walks SLOTS (K a power of two <= 16384: every attempt starts on an even word),
// k_mix_walk_any walks WORD positions (any other K <= 4095).
//
// One warp walks (a second one only helps with the prologue).  The records come from DRAM (written once by the pre-pass,
// read once) into a 1024-entry shared-memory ring by cp.async that the walker issues itself, 640 records ahead.  Per round
// the warp (1) reads 32 records from the ring, (2) looks up the current states of both replicas, (3) fetches u[i,sj],
// u[j,si] and the maintained diagonal d[k] = u[k, perm[k]], (4) evaluates log_p and the accept test, (5) resolves the
// visited chain and staleness with ballots and bit tricks, (6) commits the valid prefix: permutation + diagonal in shared
// memory and ONE coalesced store of packed (si, sj, accepted) entries into a commit log (the count matrices are built from
// the log afterwards by k_mix_count, in parallel).  Results are bit-identical to replicaexchange.py:321-349.
//
// Slots (SlotRec, or SlotRec2 in filter mode): the visited chain from slot s goes on at s+1 if log_p >= 0 (no uniform
// drawn) else at s+2, resolved with a carry-propagation bit trick.
// Words: for K that is not a power of two numba's randint rejects words (numba/_random.c: low bit_length(K-1) bits of one
// word, retried while >= K), so an attempt has no fixed length and no slot grid exists.  What stays true is that the words an
// attempt STARTING at word position p would consume for its two indices depend on the stream alone: a parallel pre-pass
// turns every position into a WordRec {i, j, len, back-mask, log of the uniform at p + len}, the window is 32 consecutive
// positions evaluated as if an attempt started at each of them, and the chain
//     next(p) = p + len(p) + (log_p(p) < 0 ? 2 : 0)
// is followed by pointer jumping over the lanes (four doublings: a hop is at least two words, so at most 16 positions of
// a window are visited).  The last < 80 words of a pass and the (astronomically rare) attempt whose indices need more than
// ANY_SCAN words are left to k_mix_walk_serial.
//
// Where the energies live (FILTER):
//   true    slots only, the tail of every pass of k_mix_walk2 (K <= 256, on its SlotRec2 records): shared memory holds a
//           24-bit floating image of every row (delta = u - rowmin as a float32 truncated to sign + 8 exponent + 15
//           mantissa bits) that gives log_p to within a RIGOROUS bound eps = 3.2e-5 * sum|delta| + tiny; the decision is
//           taken from the image, in f32, whenever it is more than eps away from both thresholds (log_p = 0 and
//           log_p = log U); a round whose committed prefix contains an undecided lane is redone with the exact f64 values
//           from L2.  The result is therefore still bit-identical.
//   false   exact f64 values from L2 every round (K > 256, or any K with RX_NO_FILTER=1).
//
// The walker's round is one dependent chain (~105 instructions); what shortens it: no f64 on the chain, no
// data-dependent branch besides the loop's (one loop condition, predicated commit), no sub-word shared stores (a
// byte-wide permutation table is slower), the absolute-to-relative lane conversion as one shift (back-mask bit order),
// and nothing re-derived from special registers inside the loop.
#pragma once

#define RING 1024         // records in the shared-memory ring
#define ANY_SCAN 40       // words scanned for the two indices of an attempt; P(more) < (1/2)^38 per attempt
#define ANY_MAX_K 4095    // 12-bit indices in the record

struct WordRec {          // 16 bytes, one per WORD position p: the attempt that would start there
    uint32_t ijl;         // i | j << 12 | len << 24; len = words that hold the two indices (0: unknown, see ANY_SCAN)
    uint32_t backmask;    // bit 31-b: the attempt at p-1-b shares a replica index with this one (or is unknown)
    double logU;          // log of the uniform made of words p+len, p+len+1: this attempt's draw if log_p < 0
};

__global__ void __launch_bounds__(256) k_words_build(const uint32_t *__restrict__ words, long long nwords, int K, uint32_t mask,
                                                     WordRec *__restrict__ rec) {
    __shared__ uint32_t s_w[256 + 31 + ANY_SCAN + 2];   // words of positions p0-31 .. p0+255+ANY_SCAN+1
    __shared__ uint32_t s_ijl[256 + 31];                 // records' first word for positions p0-31 .. p0+255
    const long long p0 = (long long)blockIdx.x * 256;
    const int t = threadIdx.x;
    for (int q = t; q < 256 + 31 + ANY_SCAN + 2; q += 256) {
        const long long p = p0 - 31 + q;
        s_w[q] = (p >= 0 && p < nwords) ? words[p] : 0u;
    }
    __syncthreads();
    for (int q = t; q < 256 + 31; q += 256) {
        const long long p = p0 - 31 + q;
        uint32_t ijl = 0;
        if (p >= 0 && p < nwords) {
            int found = 0;
            uint32_t i = 0;
            for (int k = 0; k < ANY_SCAN && p + k < nwords; k++) {
                const uint32_t r = s_w[q + k] & mask;
                if (r < (uint32_t)K) {
                    if (found == 0) { i = r; found = 1; }
                    else { ijl = i | (r << 12) | ((uint32_t)(k + 1) << 24); break; }
                }
            }
        }
        s_ijl[q] = ijl;
    }
    __syncthreads();
    const long long p = p0 + t;
    if (p >= nwords) return;
    const int q = t + 31;
    const uint32_t ijl = s_ijl[q];
    const uint32_t i = ijl & 0xfffu, j = (ijl >> 12) & 0xfffu, len = ijl >> 24;
    uint32_t bm = 0;
#pragma unroll 4
    for (int b = 0; b < 31; b++) {
        const uint32_t o = s_ijl[q - 1 - b];
        const uint32_t oi = o & 0xfffu, oj = (o >> 12) & 0xfffu;
        const bool hit = (o >> 24) == 0u || oi == i || oi == j || oj == i || oj == j;
        bm |= (hit ? 1u : 0u) << (31 - b);
    }
    WordRec r;
    r.ijl = ijl;
    r.backmask = bm;
    double lu = 0.0;
    if (len != 0u && p + len + 1 < nwords) {
        const double U = mt_double(s_w[q + len], s_w[q + len + 1]);
        lu = (U == 0.0) ? LOGU_ZERO : log(U);
    }
    r.logU = lu;
    rec[p] = r;
}

// The walker.  WORDS = false: records [ctl->head, nrec) are slots; WORDS = true: word positions (ctl->head counts words).
template <bool WORDS, bool FILTER>
__device__ __forceinline__ void ex_walk(const uint4 *__restrict__ recs, const uint32_t *__restrict__ words, unsigned nrec,
                                        const double *__restrict__ u, int K, int logK, int *__restrict__ perm_g,
                                        uint32_t *__restrict__ commit_log, const unsigned char *__restrict__ filt,
                                        const double *__restrict__ filt_rowabs, MixCtl *ctl) {
    static_assert(!(WORDS && FILTER), "the row-image filter exists for slots only");
    extern __shared__ double s_mix[];
    // layout: ring[RING] 16-byte records | diag[K] f64 | (rowabs[K]) | perm[K] i32 | (image: u16[K*K] + u8[K*K])
    uint4 *s_ring = (uint4 *)s_mix;
    double *s_diag = s_mix + 2 * RING;
    double *s_rowabs = s_diag + K;                                   // [K] |row minimum| (FILTER only)
    int *s_perm = (int *)(s_rowabs + (FILTER ? K : 0));
    unsigned char *s_q = (unsigned char *)(s_perm + K);   // 24-bit image: int16 high plane [K*K] then uint8 low plane [K*K]
    // row r, column c of the K x K matrices
    auto at = [&](unsigned r, unsigned c) { return WORDS ? r * (unsigned)K + c : (r << logK) | c; };
    // (the warp index through a shuffle: warp-uniform for the compiler, see k_mix_walk2)
    const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    for (int q = tid; q < K; q += 64) {
        const int st = perm_g[q];
        s_perm[q] = st;
        s_diag[q] = u[WORDS ? (size_t)q * K + st : ((size_t)q << logK) + st];
        // per-row share of the f64-rounding bound, f32 rounded up: 1.6e-14 (|row minimum| + 1/2)
        if (FILTER) ((float *)s_rowabs)[q] = __fmul_ru(1.6e-14f, __fadd_ru(__double2float_ru(filt_rowabs[q]), 0.5f));
    }
    if (FILTER) {
        const uint32_t *src = (const uint32_t *)filt;
        uint32_t *dst = (uint32_t *)s_q;
        for (int q = tid; q < (3 * K * K) / 4; q += 64) dst[q] = src[q];
    }
    const unsigned head0 = (unsigned)ctl->head;
    __syncthreads();
    if (warp != 0) return;   // (the second warp only helps with the prologue)

    // The records come into the ring by cp.async issued by the walker itself, 640 records ahead, topped up every 8 rounds
    // (slots) or 4 rounds (words); completion is tracked by the hardware (cp.async.wait_group), the warp barrier at the end
    // of a round makes the data visible to all lanes.  No second warp, no flags, no fences: nothing for racecheck to find.
    // (32-bit shared address through a shuffle: it then lives in a register instead of being re-derived from SR_CgaCtaId
    // every round)
    const unsigned ring_addr = __shfl_sync(0xffffffffu, (unsigned)__cvta_generic_to_shared((const void *)s_ring), 0);
    unsigned filled = head0;
    auto refill = [&](unsigned h_now) {
        while (filled < h_now + 640u && filled < nrec) {
            if (filled + (unsigned)lane < nrec)
                w2_cp_async16(ring_addr + (((filled + (unsigned)lane) & (RING - 1)) << 4), recs + (filled + lane));
            filled += 32u;
        }
        w2_cp_async_commit();
    };
    refill(head0);
    w2_cp_async_wait<0>();
    __syncwarp();

    // ---------------- walker (warp 0).  The loop is latency bound (one warp, one dependent chain per round), so it is
    // written for a short instruction stream: 32-bit indices, ring position carried from round to round.
    unsigned h = head0;
    const long long remaining0 = ctl->remaining;
    unsigned rem = remaining0 > 0x7fffffffLL ? 0x7fffffffu : (unsigned)remaining0;   // attempts this launch may still do
    const unsigned rem0 = rem;
    unsigned logpos = (unsigned)ctl->log_count, rounds = 0, slow = 0;   // the log continues where k_mix_walk2 stopped
    const unsigned lt_mask = (1u << lane) - 1u;
    const unsigned sh_amt = 32u - (unsigned)lane;
    const unsigned short *s_qhi = (const unsigned short *)s_q;            // [K*K] sign, exponent, 7 mantissa bits
    const unsigned char *s_qlo = s_q + 2 * (size_t)K * K;                  // [K*K] next 8 mantissa bits
    unsigned wpos = (h + (unsigned)lane) & (RING - 1);   // this lane's ring entry
    // words: the attempt at the window's first position has unknown indices -- k_mix_walk_serial takes over
    bool give_up = false;
    // One round.  TAIL = the launch's attempt budget may end inside the window (checked only in the last rounds).
    auto round = [&](auto tail_tag) {
        constexpr bool TAIL = decltype(tail_tag)::value;
        rounds++;
        const unsigned w = wpos;   // (h + lane) & (RING - 1), carried from round to round
        const uint4 rq = w2_lds128(ring_addr + (w << 4));
        const uint32_t backmask = rq.y;
        unsigned i, j, len = 0;
        if constexpr (WORDS) { i = rq.x & 0xfffu; j = (rq.x >> 12) & 0xfffu; len = rq.x >> 24; }
        else { i = rq.x & 0xffffu; j = rq.x >> 16; }
        const bool unknown = WORDS && len == 0u;
        // f64 log of the uniform an attempt here would draw: for a slot it belongs to the NEXT slot (words z, w of its
        // SlotRec), for a word position it is the record's own
        double logU = 0.0;
        if (!FILTER) {
            const uint2 lw = WORDS ? make_uint2(rq.z, rq.w) : w2_lds64(ring_addr + (((w + 1) & (RING - 1)) << 4) + 8u);
            logU = __hiloint2double((int)lw.y, (int)lw.x);
        }
        const int si = s_perm[i], sj = s_perm[j];
        const unsigned a_ij = at(i, (unsigned)sj), a_ji = at(j, (unsigned)si);
        bool ge0, acc, undecided = false;
        double e_ij = 0.0, e_ji = 0.0;   // exact off-diagonal values, needed by the commit (new diagonal)
        if (FILTER) {
            // image of u: 24-bit floats of delta = u - rowmin; logp~ = (d_ii - d_ij) + (d_jj - d_ji), |logp~ - logp_ref| <= eps
            const unsigned a_ii = at(i, (unsigned)si), a_jj = at(j, (unsigned)sj);
            // (hi << 16) | (lo << 8) in one byte permute
            const float f_ii = __uint_as_float(__byte_perm((unsigned)s_qhi[a_ii], (unsigned)s_qlo[a_ii], 0x1045));
            const float f_ij = __uint_as_float(__byte_perm((unsigned)s_qhi[a_ij], (unsigned)s_qlo[a_ij], 0x1045));
            const float f_jj = __uint_as_float(__byte_perm((unsigned)s_qhi[a_jj], (unsigned)s_qlo[a_jj], 0x1045));
            const float f_ji = __uint_as_float(__byte_perm((unsigned)s_qhi[a_ji], (unsigned)s_qlo[a_ji], 0x1045));
            // All in f32.  Every image value is within 2^-15 (relative) of the true delta (truncation to a 15-bit
            // mantissa + f32 rounding); the f32 additions below add at most 2^-23 of the magnitudes; the f64 rounding
            // of the reference's own three additions and of our centring is <= 64 ulp(f64) of the magnitudes.
            const float lp = (f_ii - f_ij) + (f_jj - f_ji);
            const float mag = (fabsf(f_ii) + fabsf(f_ij)) + (fabsf(f_jj) + fabsf(f_ji));
            // the guard band's 1e-9 rides in eps (a slightly wider eps for the sign test is only more conservative);
            // 1.6e-14 mag is inside the slack of 3.2e-5
            const float eps = fmaf(mag, 3.2e-5f, (((const float *)s_rowabs)[i] + ((const float *)s_rowabs)[j]) + 1e-9f);
            // log of the uniform, rounded to f32 by the producer: |lu - logU| <= 2^-24 |lu|; d carries one more rounding
            // (SlotRec2: the f32 log-uniform of the next slot is the third word of this slot's own record)
            const float lu = __uint_as_float(rq.z);
            const float d = lp - lu;
            const float mar = fmaf(fabsf(lp) + fabsf(lu), 1.3e-7f, eps);
            // |lp| > eps decides the sign of log_p, |d| > mar decides the comparison with the uniform (NaN: undecided)
            const bool dec_lp = fabsf(lp) > eps, dec_d = fabsf(d) > mar;
            // i == j: the reference's log_p is exactly 0 for finite energies (-(e+e)+e+e), accepted without a draw
            const bool same = (i == j) && (fabsf(f_ii) <= 3.0e38f);
            ge0 = (dec_lp && lp > 0.f) || same;
            acc = ge0 || (dec_lp && dec_d && d > 0.f);
            const bool decided = ge0 || (dec_lp && dec_d);
            undecided = !decided;   // resolved below, and only if the lane turns out to matter
        } else {
            e_ij = u[a_ij];
            e_ji = u[a_ji];
            const double logp = swap_logp(e_ij, e_ji, s_diag[i], s_diag[j]);
            const double d = logp - logU;
            ge0 = logp >= 0.0;
            acc = ge0 || d > 1e-9;
            const bool ambiguous = !ge0 && fabs(d) <= 1e-9 && !unknown;   // NaN compares false: rejected, like the reference
            if (__any_sync(0xffffffffu, ambiguous)) {
                if (ambiguous) {  // too close to call in the log domain: do exactly what the reference does
                    const size_t a = WORDS ? (size_t)h + lane + len : 2 * (size_t)(h + lane + 1);   // the uniform's words
                    acc = mt_double(words[a], words[a + 1]) < rx_exp_cr(logp);
                    slow++;
                }
            }
        }
        unsigned V, C, low, cm, n, advance;
        auto resolve = [&]() {
            unsigned full;   // how far the window advances if all of it commits
            [[maybe_unused]] const unsigned G = WORDS ? 0u : __ballot_sync(0xffffffffu, ge0);   // (slots)
            const unsigned A = __ballot_sync(0xffffffffu, acc && i != j && !unknown);   // accepted and really changing the permutation
            if constexpr (WORDS) {
                // Pointer jumping over the lanes: N = window position of the attempt after this one (>= 32: beyond the
                // window), R = set of positions the chain from here visits; lane 0 holds the chain from h.
                unsigned N = unknown ? 64u : (unsigned)lane + len + (ge0 ? 0u : 2u);
                unsigned R = 1u << lane;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const unsigned src = N & 31u;
                    const unsigned Rn = __shfl_sync(0xffffffffu, R, src), Nn = __shfl_sync(0xffffffffu, N, src);
                    if (N < 32u) { R |= Rn; N = Nn; }
                }
                V = __shfl_sync(0xffffffffu, R, 0);
                full = __shfl_sync(0xffffffffu, N, 0);
            } else {
                // Visited chain: from a visited slot s the next attempt starts at s+1 if log_p >= 0 (no uniform drawn) else
                // at s+2.  skip[s+1] = NG[s] & ~skip[s]: inside a run of NG ones the skip flag alternates, so skip[s] =
                // parity of (s - run start); runs are split by the parity of their start with an add-carry (32-bit adds +
                // carry out).
                const unsigned X = ~G;
                const unsigned starts = X & ~(X << 1);
                const unsigned SE = starts & 0x55555555u, SO = starts & 0xAAAAAAAAu;
                const unsigned sumE = X + SE, sumO = X + SO;
                const unsigned skip = (((sumE ^ X) & ~SE) & 0xAAAAAAAAu) | (((sumO ^ X) & ~SO) & 0x55555555u);
                V = ~skip;
                // bit 32 (even position) of the skip word can only be set by the carry of an odd-start run
                full = 32u + (sumO < X ? 1u : 0u);
            }
            const unsigned VA = V & A;  // visited, accepted, really changing the permutation
            // lane t is stale if an earlier visited state-changing swap in this window shares a replica with it
            unsigned earlier;   // bit 31-b: lane t-1-b is a visited state-changing swap (shl by 32 gives 0 for lane 0)
            asm("shl.b32 %0, %1, %2;" : "=r"(earlier) : "r"(VA), "r"(sh_amt));
            C = __ballot_sync(0xffffffffu, (earlier & backmask) != 0u || unknown) & V;
            low = C & (0u - C);
            cm = V & (low - 1u);           // low == 0 -> all lanes
            n = __popc(cm);
            advance = C ? (unsigned)__popc(low - 1u) : full;
        };
        if constexpr (FILTER) {
            // The filter's undecided lanes carry arbitrary ge0/acc.  Bits of V, C and cm below the lowest undecided
            // visited lane do not depend on them (the chain and the staleness test only look downwards), so the round
            // is resolved speculatively and redone with exact values only when such a lane lies inside the committed
            // prefix -- the ballot of the undecided lanes is off the critical path and rarely matters.
            const unsigned U = __ballot_sync(0xffffffffu, undecided);
            resolve();
            if (U & cm) {
                if (undecided) {   // exact path for this lane: the f64 values from L2
                    const unsigned d = w2_exact_decision(u, K, rq.x, (unsigned)si, (unsigned)sj, words, 2 * (size_t)(h + lane + 1));
                    ge0 = (d & 1u) != 0u;
                    acc = (d & 2u) != 0u;
                    slow++;
                }
                resolve();
            }
        } else {
            resolve();
        }
        if (WORDS && (C & 1u)) { give_up = true; return; }   // (only an unknown position can stop the window's first attempt)
        if (TAIL && n > rem) {
            unsigned pos = 0;  // the first visited lane we must NOT run: the (rem+1)-th set bit of cm
            for (unsigned cnt = 0; pos < 32; pos++)
                if ((cm >> pos) & 1u) { if (cnt == rem) break; cnt++; }
            cm &= (1u << pos) - 1u;
            n = rem;
            advance = pos;
        }
        // commit: everything is computed by every lane, only the stores are predicated (no divergent block); bit 31 marks
        // a logged attempt (the count kernel also reads the filter walkers' sparse log)
        const bool mine = (cm >> lane) & 1u;
        const unsigned log_at = logpos + __popc(cm & lt_mask);
        const uint32_t entry = (uint32_t)si | ((uint32_t)sj << LOG_STATE_BITS) | (acc ? (1u << 31) | (1u << LOG_ACC_BIT) : (1u << 31));
        const bool swaps = mine && acc && i != j;  // an i == j lane must not write: a later committed lane may swap this replica
        if (mine) commit_log[log_at] = entry;
        if (swaps) { s_perm[i] = sj; s_perm[j] = si; }
        if (!FILTER) { if (swaps) { s_diag[i] = e_ij; s_diag[j] = e_ji; } }   // the image needs no f64 diagonal
        logpos += n;
        h += advance;
        wpos = (wpos + advance) & (RING - 1);
        rem -= n;
        // Every R rounds top the ring up to 640 records ahead and wait for all copies but the ones just issued.  A round
        // advances by at most 33 slots, or 31 + ANY_SCAN + 2 = 73 words.  The next R rounds read below h + 33 R + 32
        // (slots) / h + 73 R + 32 (words); the copies already waited for were issued at the previous top-up, at most R
        // rounds back, and reach h - 33 R + 640 / h - 73 R + 640.  So 2 R 33 + 32 <= 640 and 2 R 73 + 32 <= 640: R = 8 for
        // slots (the next 8 rounds read below h + 296, the copies reach h + 376), R = 4 for words (below h + 324, h + 348).
        if ((rounds & (WORDS ? 3u : 7u)) == 0u) { refill(h); w2_cp_async_wait<1>(); }
        __syncwarp();
    };
    // a round may start while every attempt of its window has its records (slots: and the next slot's uniform), words: its
    // index words and its uniform inside the pass
    const unsigned span = WORDS ? 32u + ANY_SCAN + 2u : 33u;
    while (rem > 0 && h + span <= nrec && !give_up) {
        if (rem >= 33) {
            // main loop: a round commits at most 32 attempts, so the budget cannot end inside it
            do { round(std::false_type()); } while (rem >= 33u && h + span <= nrec && !give_up);
        } else {
            round(std::true_type());
        }
    }
    w2_cp_async_wait<0>();
    for (int q = lane; q < K; q += 32) perm_g[q] = s_perm[q];
    slow = __reduce_add_sync(0xffffffffu, slow);
    if (lane == 0) {
        const long long remaining = remaining0 - (long long)(rem0 - rem);
        ctl->head = h;
        ctl->remaining = remaining;
        ctl->status = remaining > 0 ? 1 : 0;
        ctl->rounds += (int)rounds;
        ctl->slow_exp += slow;
        ctl->log_count = logpos;
    }
}

// FILTER: on the 24-bit image, over the SlotRec2 records of k_mix_walk2 (the tail of its passes); otherwise f64 from L2
template <bool FILTER>
__global__ void __launch_bounds__(64) k_mix_walk_pow2(const SlotRec *__restrict__ rec, const uint32_t *__restrict__ words,
                                                      unsigned nslots, const double *__restrict__ u, int K, int logK,
                                                      int *__restrict__ perm_g, uint32_t *__restrict__ commit_log,
                                                      const unsigned char *__restrict__ filt,
                                                      const double *__restrict__ filt_rowabs, MixCtl *ctl) {
    ex_walk<false, FILTER>((const uint4 *)rec, words, nslots, u, K, logK, perm_g, commit_log, filt, filt_rowabs, ctl);
}

__global__ void __launch_bounds__(64) k_mix_walk_any(const WordRec *__restrict__ rec, const uint32_t *__restrict__ words,
                                                     unsigned nwords, const double *__restrict__ u, int K,
                                                     int *__restrict__ perm_g, uint32_t *__restrict__ commit_log, MixCtl *ctl) {
    ex_walk<true, false>((const uint4 *)rec, words, nwords, u, K, 0, perm_g, commit_log, nullptr, nullptr, ctl);
}
