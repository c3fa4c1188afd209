// rx_walk2c.cuh -- candidate coordinates for the filter walker k_mix_walk2c (rx_walk2.cuh) at any K <= 256 and the exact
// walker k_mix_walk_cand (rx_walk_exact.cuh) at any K <= ANY_MAX_K (included by rx_mix.cu after rx_walk2.cuh).
//
// For K that is not a power of two numba's randint rejects words (numba/_random.c: low bit_length(K-1) bits of one word,
// retried while >= K), so attempts have no fixed length in the word stream.  In CANDIDATE coordinates they do: let the
// candidates be the words whose masked value is < K, numbered c = 0, 1, ... in stream order.  An attempt that starts with
// candidate c as its next unconsumed candidate takes i = cand[c], j = cand[c+1], whatever rejected words lie in between;
// if log_p >= 0 the next attempt starts at candidate c+2; otherwise the uniform is made of the two RAW words that follow
// candidate c+1, and the next attempt starts at c + 2 + k, where k in {0, 1, 2} counts the candidates among those two
// words -- a property of the stream alone.  So a state-independent pre-pass (flag, scan, scatter, records) gives one
// 16-byte record per candidate index {i | j << 16, back-mask, f32 log-uniform of this attempt, k}, and the walker is
// the one of k_mix_walk2 with a window of 32 candidate indices and hops of 2, 3 or 4 instead of 1 or 2 (its visited chain:
// w2_chain_cand; replicaexchange.py:321-349 bit for bit, like every other walker here).  The exact walker takes a CandRec
// per candidate index instead, with the f64 log-uniform and 12-bit indices.
#pragma once

#define CAND_TILE 2048    // words per block of the flag/scan/scatter pre-pass
#define ANY_MAX_K 4095    // 12-bit indices in a CandRec

struct CandRec {          // 16 bytes, one per candidate index c: the attempt that would start there (exact walker)
    uint32_t ijk;         // i | j << 12 | k << 24; k = hop class as in SlotRec2
    uint32_t backmask;    // bit 31-b: the attempt at c-1-b shares a replica index with this one
    double logU;          // log of the uniform this attempt draws if log_p < 0
};

// (1) candidates per tile of CAND_TILE words
__global__ void __launch_bounds__(256) k_cand_count(const uint32_t *__restrict__ words, long long nwords, int K, uint32_t mask,
                                                    uint32_t *__restrict__ tile_count) {
    __shared__ uint32_t s_c[8];
    const long long p0 = (long long)blockIdx.x * CAND_TILE;
    uint32_t n = 0;
    for (int q = threadIdx.x; q < CAND_TILE; q += 256) {
        const long long p = p0 + q;
        if (p < nwords && (words[p] & mask) < (uint32_t)K) n++;
    }
    n = __reduce_add_sync(0xffffffffu, n);
    if ((threadIdx.x & 31) == 0) s_c[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int q = 0; q < 8; q++) t += s_c[q];
        tile_count[blockIdx.x] = t;
    }
}

// (2) exclusive scan of the tile counts in place (one block; ntiles <= 2^25 / CAND_TILE), total to *ncand
__global__ void __launch_bounds__(1024) k_cand_scan(uint32_t *__restrict__ tile_count, int ntiles, uint32_t *__restrict__ ncand) {
    __shared__ uint32_t s_part[1024];
    const int t = threadIdx.x;
    const int per = (ntiles + 1023) / 1024;
    const int lo = t * per, hi = min(lo + per, ntiles);
    uint32_t sum = 0;
    for (int q = lo; q < hi; q++) sum += tile_count[q];
    s_part[t] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {   // Hillis-Steele inclusive scan of the 1024 partial sums
        const uint32_t v = t >= o ? s_part[t - o] : 0u;
        __syncthreads();
        s_part[t] += v;
        __syncthreads();
    }
    uint32_t run = s_part[t] - sum;   // exclusive prefix of this thread's range
    for (int q = lo; q < hi; q++) { const uint32_t c = tile_count[q]; tile_count[q] = run; run += c; }
    if (t == 1023) *ncand = s_part[1023];
}

// (3) word position of every candidate: cpos[c]
__global__ void __launch_bounds__(256) k_cand_scatter(const uint32_t *__restrict__ words, long long nwords, int K, uint32_t mask,
                                                      const uint32_t *__restrict__ tile_base, uint32_t *__restrict__ cpos) {
    __shared__ uint32_t s_w[8];
    const long long p0 = (long long)blockIdx.x * CAND_TILE;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    // thread t owns the 8 consecutive words p0 + 8 t .. p0 + 8 t + 7
    uint32_t flags = 0;
    for (int q = 0; q < 8; q++) {
        const long long p = p0 + 8 * t + q;
        if (p < nwords && (words[p] & mask) < (uint32_t)K) flags |= 1u << q;
    }
    const uint32_t mine = (uint32_t)__popc(flags);
    uint32_t incl = mine;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t base = tile_base[blockIdx.x];
    for (int q = 0; q < warp; q++) base += s_w[q];
    uint32_t c = base + incl - mine;
    for (int q = 0; q < 8; q++)
        if ((flags >> q) & 1u) cpos[c++] = (uint32_t)(p0 + 8 * t + q);
}

// (4) one record per candidate index c < ncand - 3 (the attempt that would start there): SlotRec2 for the filter walker,
// CandRec (EXACT) for the exact walker
template <bool EXACT>
__global__ void __launch_bounds__(256) k_cand_records(const uint32_t *__restrict__ words, const uint32_t *__restrict__ cpos,
                                                      const uint32_t *__restrict__ ncand_p, uint32_t mask,
                                                      std::conditional_t<EXACT, CandRec, SlotRec2> *__restrict__ rec) {
    __shared__ uint32_t s_v[256 + 31 + 1];   // values of candidates c0-31 .. c0+256
    const uint32_t ncand = *ncand_p;
    const long long c0 = (long long)blockIdx.x * 256;
    if (c0 >= (long long)ncand) return;
    const int t = threadIdx.x;
    for (int q = t; q < 256 + 32; q += 256) {
        const long long c = c0 - 31 + q;
        s_v[q] = (c >= 0 && c < (long long)ncand) ? (words[cpos[c]] & mask) : 0xffffu;
    }
    __syncthreads();
    const long long c = c0 + t;
    if (c + 3 >= (long long)ncand) return;
    const int q = t + 31;
    const uint32_t i = s_v[q], j = s_v[q + 1];
    uint32_t bm = 0;
#pragma unroll 4
    for (int b = 0; b < 31; b++) {   // the attempt at c-1-b takes the candidates c-1-b and c-b
        const uint32_t oi = s_v[q - 1 - b], oj = s_v[q - b];
        const bool hit = (c - 1 - b >= 0) && (oi == i || oi == j || oj == i || oj == j);
        bm |= (hit ? 1u : 0u) << (31 - b);
    }
    const uint32_t a = cpos[c + 1] + 1u;   // the uniform's words: a, a + 1 (cpos[c+3] >= a + 1: inside the stream)
    const uint32_t k = (cpos[c + 2] <= a + 1u ? 1u : 0u) + (cpos[c + 3] <= a + 1u ? 1u : 0u);
    const double U = mt_double(words[a], words[a + 1]);
    if constexpr (EXACT) {
        CandRec r;
        r.ijk = i | (j << 12) | (k << 24);
        r.backmask = bm;
        r.logU = (U == 0.0) ? LOGU_ZERO : log(U);
        rec[c] = r;
    } else {
        SlotRec2 r;
        r.ij = i | (j << 16);
        r.backmask = bm;
        r.lu_next = __float_as_uint((float)((U == 0.0) ? LOGU_ZERO : log(U)));
        r.k = k;
        rec[c] = r;
    }
}
