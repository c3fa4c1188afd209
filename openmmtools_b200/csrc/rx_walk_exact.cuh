// rx_walk_exact.cuh -- the exact speculative swap-all walker (included by rx_mix.cu after rx_walk2c.cuh).  One body, two
// coordinate systems: k_mix_walk_pow2 walks SLOTS (K a power of two <= 16384: every attempt starts on an even word),
// k_mix_walk_cand walks CANDIDATE indices (any other K <= ANY_MAX_K, rx_walk2c.cuh).
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
// Candidates (CandRec {i | j << 12 | k << 24, back-mask, f64 log U of the attempt}, k_cand_records<true>): the chain goes on
// at c+2 if log_p >= 0, else at c+2+k, resolved by w2_chain_cand; a visited position whose hop would leave the window is a
// forced stop that opens the next round, so a round advances by at most 32 records.  The pass starts at candidate 0; the
// last < 35 candidates of a pass are left to k_mix_walk_serial, which continues from the word position reported in
// ctl->head: the next attempt's first candidate, or the word after the last attempt if the budget ended in the walker.
//
// Where the energies live (FILTER):
//   true    slots only, the tail of every pass of k_mix_walk2 (K <= 256, on its SlotRec2 records): shared memory holds a
//           24-bit floating image of every row (delta = u - rowmin as a float32 truncated to sign + 8 exponent + 15
//           mantissa bits) that gives log_p to within a RIGOROUS bound eps = 3.2e-5 * sum|delta| + tiny; the decision is
//           taken from the image, in f32, whenever it is more than eps away from both thresholds (log_p = 0 and
//           log_p = log U); a round whose committed prefix contains an undecided lane is redone with the exact f64 values
//           from L2.  The result is therefore still bit-identical.
//   false   exact f64 values from L2 every round (slots: K > 256, or any K with RX_NO_FILTER=1; every candidate walk).
//
// The walker's round is one dependent chain (~105 instructions); what shortens it: no f64 on the chain, no
// data-dependent branch besides the loop's (one loop condition, predicated commit), no sub-word shared stores (a
// byte-wide permutation table is slower), the absolute-to-relative lane conversion as one shift (back-mask bit order),
// and nothing re-derived from special registers inside the loop.
#pragma once

#define RING 1024         // records in the shared-memory ring

// The walker.  CAND = false: records [ctl->head, nrec) are slots; CAND = true: candidate indices [0, nrec), cpos gives the
// word position of every candidate (ctl->head counts words).
template <bool CAND, bool FILTER>
__device__ __forceinline__ void ex_walk(const uint4 *__restrict__ recs, const uint32_t *__restrict__ words,
                                        const uint32_t *__restrict__ cpos, unsigned nrec, const double *__restrict__ u, int K,
                                        int logK, int *__restrict__ perm_g, uint32_t *__restrict__ commit_log,
                                        const unsigned char *__restrict__ filt, const double *__restrict__ filt_rowabs,
                                        MixCtl *ctl) {
    static_assert(!(CAND && FILTER), "the row-image filter of this walker exists for slots only");
    extern __shared__ double s_mix[];
    // layout: ring[RING] 16-byte records | diag[K] f64 | (rowabs[K]) | perm[K] i32 | (image: u16[K*K] + u8[K*K])
    uint4 *s_ring = (uint4 *)s_mix;
    double *s_diag = s_mix + 2 * RING;
    double *s_rowabs = s_diag + K;                                   // [K] |row minimum| (FILTER only)
    int *s_perm = (int *)(s_rowabs + (FILTER ? K : 0));
    unsigned char *s_q = (unsigned char *)(s_perm + K);   // 24-bit image: int16 high plane [K*K] then uint8 low plane [K*K]
    // row r, column c of the K x K matrices
    auto at = [&](unsigned r, unsigned c) { return CAND ? r * (unsigned)K + c : (r << logK) | c; };
    // (the warp index through a shuffle: warp-uniform for the compiler, see k_mix_walk2)
    const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    for (int q = tid; q < K; q += 64) {
        const int st = perm_g[q];
        s_perm[q] = st;
        s_diag[q] = u[CAND ? (size_t)q * K + st : ((size_t)q << logK) + st];
        // per-row share of the f64-rounding bound, f32 rounded up: 1.6e-14 (|row minimum| + 1/2)
        if (FILTER) ((float *)s_rowabs)[q] = __fmul_ru(1.6e-14f, __fadd_ru(__double2float_ru(filt_rowabs[q]), 0.5f));
    }
    if (FILTER) {
        const uint32_t *src = (const uint32_t *)filt;
        uint32_t *dst = (uint32_t *)s_q;
        for (int q = tid; q < (3 * K * K) / 4; q += 64) dst[q] = src[q];
    }
    // slots: the pass continues at slot ctl->head; candidates: a pass starts at candidate 0 (word position ctl->head == 0)
    const unsigned head0 = CAND ? 0u : (unsigned)ctl->head;
    __syncthreads();
    if (warp != 0) return;   // (the second warp only helps with the prologue)

    // The records come into the ring by cp.async issued by the walker itself, 640 records ahead, topped up every 8 rounds;
    // completion is tracked by the hardware (cp.async.wait_group), the warp barrier at the end of a round makes the data
    // visible to all lanes.  No second warp, no flags, no fences: nothing for racecheck to find.
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
    // candidates: the word after the last attempt, when the budget ends in the walker (the plain loop then has nothing to
    // do, and the stream position must be the reference's)
    [[maybe_unused]] unsigned end_word = 0;
    // One round.  TAIL = the launch's attempt budget may end inside the window (checked only in the last rounds).
    auto round = [&](auto tail_tag) {
        constexpr bool TAIL = decltype(tail_tag)::value;
        rounds++;
        const unsigned w = wpos;   // (h + lane) & (RING - 1), carried from round to round
        const uint4 rq = w2_lds128(ring_addr + (w << 4));
        const uint32_t backmask = rq.y;
        unsigned i, j;
        [[maybe_unused]] unsigned K1 = 0, K2 = 0;   // candidates: ballots of the hop classes k == 1, k == 2 (state independent)
        if constexpr (CAND) {
            i = rq.x & 0xfffu; j = (rq.x >> 12) & 0xfffu;
            K1 = __ballot_sync(0xffffffffu, (rq.x >> 24) == 1u);
            K2 = __ballot_sync(0xffffffffu, (rq.x >> 24) == 2u);
        } else {
            i = rq.x & 0xffffu; j = rq.x >> 16;
        }
        // f64 log of the uniform an attempt here would draw: for a slot it belongs to the NEXT slot (words z, w of its
        // SlotRec), for a candidate index it is the record's own
        double logU = 0.0;
        if (!FILTER) {
            const uint2 lw = CAND ? make_uint2(rq.z, rq.w) : w2_lds64(ring_addr + (((w + 1) & (RING - 1)) << 4) + 8u);
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
            const bool ambiguous = !ge0 && fabs(d) <= 1e-9;   // NaN compares false: rejected, like the reference
            if (__any_sync(0xffffffffu, ambiguous)) {
                if (ambiguous) {  // too close to call in the log domain: do exactly what the reference does
                    const size_t a = CAND ? (size_t)cpos[h + lane + 1] + 1 : 2 * (size_t)(h + lane + 1);   // the uniform's words
                    acc = mt_double(words[a], words[a + 1]) < rx_exp_cr(logp);
                    slow++;
                }
            }
        }
        unsigned V, C, low, cm, n, advance;
        auto resolve = [&]() {
            unsigned full;   // how far the window advances if all of it commits
            unsigned Cf = 0;   // candidates: forced stops, visited positions whose hop would leave the window
            const unsigned G = __ballot_sync(0xffffffffu, ge0);
            const unsigned A = __ballot_sync(0xffffffffu, acc && i != j);   // accepted and really changing the permutation
            if constexpr (CAND) {
                w2_chain_cand(G, K1, K2, V, Cf);
                full = 32u;
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
            // the stops: stale visited lanes and forced stops (never position 0)
            C = (__ballot_sync(0xffffffffu, (earlier & backmask) != 0u) | Cf) & V;
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
        if (TAIL && n > rem) {
            unsigned pos = 0;  // the first visited lane we must NOT run: the (rem+1)-th set bit of cm
            for (unsigned cnt = 0; pos < 32; pos++)
                if ((cm >> pos) & 1u) { if (cnt == rem) break; cnt++; }
            cm &= (1u << pos) - 1u;
            n = rem;
            advance = pos;
        }
        if constexpr (CAND) {
            if (TAIL && n == rem) {   // the budget ends in this round: the word after its last attempt (i, j, uniform?)
                const unsigned last = 31u - __clz(cm);
                end_word = __shfl_sync(0xffffffffu, cpos[h + lane + 1] + (ge0 ? 1u : 3u), last);
            }
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
        // advances by at most 33 slots or 32 candidates.  The next R rounds read below h + 33 R + 32; the copies already
        // waited for were issued at the previous top-up, at most R rounds back, and reach h - 33 R + 640.  So
        // 2 R 33 + 32 <= 640: R = 8 (the next 8 rounds read below h + 296, the copies reach h + 376).
        if ((rounds & 7u) == 0u) { refill(h); w2_cp_async_wait<1>(); }
        __syncwarp();
    };
    // a round may start while every attempt of its window has its record (slots: and the next slot's uniform)
    const unsigned span = CAND ? 32u : 33u;
    while (rem > 0 && h + span <= nrec) {
        if (rem >= 33) {
            // main loop: a round commits at most 32 attempts, so the budget cannot end inside it
            do { round(std::false_type()); } while (rem >= 33u && h + span <= nrec);
        } else {
            round(std::true_type());
        }
    }
    w2_cp_async_wait<0>();
    for (int q = lane; q < K; q += 32) perm_g[q] = s_perm[q];
    slow = __reduce_add_sync(0xffffffffu, slow);
    if (lane == 0) {
        const long long remaining = remaining0 - (long long)(rem0 - rem);
        if constexpr (!CAND) ctl->head = h;
        else if (h > 0) ctl->head = rem ? (long long)cpos[h] : (long long)end_word;   // word position for the plain loop
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
    ex_walk<false, FILTER>((const uint4 *)rec, words, nullptr, nslots, u, K, logK, perm_g, commit_log, filt, filt_rowabs, ctl);
}

__global__ void __launch_bounds__(64) k_mix_walk_cand(const CandRec *__restrict__ rec, const uint32_t *__restrict__ words,
                                                      const uint32_t *__restrict__ cpos, const uint32_t *__restrict__ ncand_p,
                                                      const double *__restrict__ u, int K, int *__restrict__ perm_g,
                                                      uint32_t *__restrict__ commit_log, MixCtl *ctl) {
    const unsigned ncand = *ncand_p;   // records exist for c < ncand - 3
    ex_walk<true, false>((const uint4 *)rec, words, cpos, ncand >= 3u ? ncand - 3u : 0u, u, K, 0, perm_g, commit_log, nullptr,
                         nullptr, ctl);
}
