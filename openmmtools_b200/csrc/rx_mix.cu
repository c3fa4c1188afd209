// rx_mix.cu -- replica mixing (Gibbs / Metropolis state swaps) on the device.
//
// Replaces ReplicaExchangeSampler._mix_replicas (openmmtools/multistate/replicaexchange.py:255-292):
//   swap-all       _mix_all_replicas_numba  (replicaexchange.py:294-349)  -> k_mix_walk2 / k_mix_walk_pow2 (K a power of two),
//                                                                            k_mix_walk2c / k_mix_walk_cand (any other K), k_mix_walk_serial
//   swap-neighbors _mix_neighboring_replicas (replicaexchange.py:366-406) -> k_mix_neighbors
// The results are bit-identical to the reference for the same MT19937 state: the random stream is numba's
// (numba/_random.c:37-73; randint = low bit_length(K-1) bits of one word with rejection, rand = 53-bit double
// from two words), reproduced on the device by k_mt_generate.
//
// Design (see DESIGN.md "mixing"): the K^3-long chain is data dependent (an attempt draws rand() only when
// log_p < 0), but the stream itself is state independent.  For power-of-two K every attempt starts on an
// even word ("slot"), so a parallel pre-pass turns the stream into slot records (i, j, log U, overlap mask)
// and ONE warp then walks the chain speculatively: 32 lanes evaluate 32 consecutive slots under the current
// permutation, the visited-slot chain is resolved with a carry-propagation bit trick, and the longest prefix
// in which no visited slot touches a replica swapped earlier in the same window is committed.  Any other K is walked the
// same way in candidate coordinates (the words randint accepts, rx_walk2c.cuh).  One plan per call (mix_plan) chooses the
// walkers: the filter walkers (rx_walk2.cuh) take the bulk of a pass for K <= 256 unless RX_NO_FILTER=1; the exact walker
// (rx_walk_exact.cuh) finishes their passes over slots and takes their place in either coordinate system for larger K; the
// plain loop k_mix_walk_serial finishes every pass over candidates and walks every K that has no walker.
#include "rx_internal.cuh"
#include <type_traits>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <chrono>
static inline double rx_wall_us() { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// ------------------------------------------------------------------------------------------------------
// MT19937 generation: x[n+624] = x[n+397] ^ twist(x[n], x[n+1]); 227 words are independent per step and
// a thread's second consecutive step only needs its own previous output, so there is one barrier per 454
// words.  `window` holds the last 624 raw words and is advanced by exactly n.
// ------------------------------------------------------------------------------------------------------
#define MT_RING 2048

__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}
__device__ __forceinline__ uint32_t mt_twist(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return c ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

__global__ void __launch_bounds__(256) k_mt_generate(uint32_t *__restrict__ window, uint32_t *__restrict__ out,
                                                     long long n) {
    __shared__ uint32_t buf[MT_RING];
    const int t = threadIdx.x;
    for (int q = t; q < 624; q += 256) buf[q] = window[q];
    __syncthreads();
    long long produced = 0;
    unsigned base = 0;
    while (produced < n) {
        if (t < 227) {
            uint32_t a = buf[(base + t) & (MT_RING - 1)], b = buf[(base + t + 1) & (MT_RING - 1)];
            uint32_t c = buf[(base + t + 397) & (MT_RING - 1)];
            uint32_t x = mt_twist(a, b, c);
            buf[(base + t + 624) & (MT_RING - 1)] = x;
            if (out && produced + t < n) out[produced + t] = mt_temper(x);
            // second step: x[n+227+t+624] needs x[n+227+t], x[n+228+t] (old) and this thread's x[n+624+t]
            a = buf[(base + 227 + t) & (MT_RING - 1)];
            b = buf[(base + 228 + t) & (MT_RING - 1)];
            uint32_t x2 = mt_twist(a, b, x);
            buf[(base + 227 + t + 624) & (MT_RING - 1)] = x2;
            if (out && produced + 227 + t < n) out[produced + 227 + t] = mt_temper(x2);
        }
        __syncthreads();
        produced += 454;
        base += 454;
    }
    // ring position of x_{n0 + n}: base - (produced - n)
    unsigned w0 = base - (unsigned)(produced - n);
    __syncthreads();
    uint32_t keep[3];
    for (int q = t, m = 0; q < 624; q += 256, m++) keep[m] = buf[(w0 + q) & (MT_RING - 1)];
    for (int q = t, m = 0; q < 624; q += 256, m++) window[q] = keep[m];
}

__global__ void k_copy_words(const uint32_t *__restrict__ src, uint32_t *__restrict__ dst, long long n) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) dst[i] = src[i];
}

// numba/numpy double from two words: ((a >> 5) * 2^26 + (b >> 6)) / 2^53
__device__ __forceinline__ double mt_double(uint32_t w0, uint32_t w1) {
    return ((double)(w0 >> 5) * 67108864.0 + (double)(w1 >> 6)) * (1.0 / 9007199254740992.0);
}

// log_p exactly as the reference evaluates it: -(e_ij + e_ji) + e_ii + e_jj, left to right, no contraction.
__device__ __forceinline__ double swap_logp(double e_ij, double e_ji, double e_ii, double e_jj) {
    return __dadd_rn(__dadd_rn(-__dadd_rn(e_ij, e_ji), e_ii), e_jj);
}

// exp(x), correctly rounded (round to nearest) -- for the reference's own test `rand() < exp(log_p)` in the cases where
// it is not decided in the log domain.  CUDA's exp() may be off by one ulp; the host libm the reference calls (numba -> libm
// exp) is correctly rounded at all but ~1 % of the arguments: with a one-ulp error the decision differs from the
// reference's whenever U is the double next to exp(log_p) (tests/test_gpu_mixing.py constructs such matrices).
// Double-double evaluation: x = k ln2 + r (three-part ln 2, the first part fdlibm's ln2HI so that k ln2HI is exact),
// expm1(r / 256) by its Taylor series to the 9th power, eight squarings in the form m <- m (m + 2), result (1 + m) 2^k;
// relative error ~2^-95, so the rounding can only be wrong if exp(x) lies within ~2^-40 ulp of a midpoint between two doubles.
// Rare path only (guard band, plain loop): its speed is irrelevant.
struct rx_dd { double hi, lo; };
__device__ __forceinline__ rx_dd dd_fast_two_sum(double a, double b) {
    const double s = __dadd_rn(a, b);
    return {s, __dadd_rn(b, -__dadd_rn(s, -a))};
}
__device__ __forceinline__ rx_dd dd_two_sum(double a, double b) {
    const double s = __dadd_rn(a, b), bb = __dadd_rn(s, -a);
    return {s, __dadd_rn(__dadd_rn(a, -__dadd_rn(s, -bb)), __dadd_rn(b, -bb))};
}
__device__ __forceinline__ rx_dd dd_add(rx_dd a, rx_dd b) {
    rx_dd s = dd_two_sum(a.hi, b.hi);
    const rx_dd t = dd_two_sum(a.lo, b.lo);
    s = dd_fast_two_sum(s.hi, __dadd_rn(s.lo, t.hi));
    return dd_fast_two_sum(s.hi, __dadd_rn(s.lo, t.lo));
}
__device__ __forceinline__ rx_dd dd_mul(rx_dd a, rx_dd b) {
    const double p = __dmul_rn(a.hi, b.hi);
    double e = __fma_rn(a.hi, b.hi, -p);
    e = __fma_rn(a.hi, b.lo, e);
    e = __fma_rn(a.lo, b.hi, e);
    return dd_fast_two_sum(p, e);
}
__device__ __noinline__ double rx_exp_cr(double x) {
    if (!(x == x)) return x;
    if (x > 709.782712893384) return INFINITY;
    if (x < -745.1332191019412) return 0.0;      // exp(x) <= 2^-1075 rounds to zero
    const double kd = rint(__dmul_rn(x, 1.4426950408889634));
    const double ln2HI = 6.93147180369123816490e-01, ln2LO = 1.9082149292705877e-10, ln2LL = 1.1612227229362532e-26;
    const double r0 = __fma_rn(-kd, ln2HI, x);                  // exact
    const double p = __dmul_rn(kd, ln2LO), pe = __fma_rn(kd, ln2LO, -p);
    rx_dd r = dd_two_sum(r0, -p);
    r = dd_fast_two_sum(r.hi, __dadd_rn(r.lo, -__dadd_rn(pe, __dmul_rn(kd, ln2LL))));
    const rx_dd s = {__dmul_rn(r.hi, 0.00390625), __dmul_rn(r.lo, 0.00390625)};   // r / 256, exact
    const rx_dd c[8] = {   // 1/2! .. 1/9!
        {0.5, 0.0},
        {0.16666666666666666, 9.25185853854297e-18},
        {0.041666666666666664, 2.3129646346357427e-18},
        {0.008333333333333333, 1.1564823173178714e-19},
        {0.001388888888888889, -5.300543954373577e-20},
        {0.0001984126984126984, 1.7209558293420705e-22},
        {2.48015873015873e-05, 2.1511947866775882e-23},
        {2.7557319223985893e-06, -1.858393274046472e-22}};
    rx_dd acc = c[7];
#pragma unroll
    for (int n = 6; n >= 0; n--) acc = dd_add(c[n], dd_mul(s, acc));
    rx_dd m = dd_add(s, dd_mul(dd_mul(s, s), acc));                  // expm1(r / 256)
#pragma unroll
    for (int q = 0; q < 8; q++) m = dd_mul(m, dd_add(m, rx_dd{2.0, 0.0}));     // expm1(2 t) = expm1(t) (expm1(t) + 2)
    const rx_dd y = dd_add(rx_dd{1.0, 0.0}, m);
    return ldexp(y.hi, (int)kd);
}

__global__ void k_selftest_exp(const double *__restrict__ x, double *__restrict__ y, int n) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) y[t] = rx_exp_cr(x[t]);
}
int rxi_selftest_exp(rx_engine *h, const double *x, double *y, int n) {
    DevBuf<double> d;
    if (n <= 0) return RX_OK;
    RX_CHECK_CUDA(h, d.alloc(2 * (size_t)n));
    RX_CHECK_CUDA(h, cudaMemcpy(d, x, (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
    k_selftest_exp<<<(n + 127) / 128, 128, 0, h->stream>>>(d, d + n, n);
    RX_CHECK_CUDA(h, cudaGetLastError());
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(y, d + n, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
    return RX_OK;
}

// ------------------------------------------------------------------------------------------------------
// The speculative chain walkers: the filter walkers (rx_walk2.cuh, rx_walk2c.cuh) and the exact walker
// (rx_walk_exact.cuh).  Their state-independent records (slot records: k_slots_build, rx_walk2.cuh; candidate records:
// k_cand_*, rx_walk2c.cuh) are built in parallel; each logs the attempts it commits as packed (si, sj, accepted) entries,
// bit 31 set.
// ------------------------------------------------------------------------------------------------------
#define LOGU_ZERO (-745.5)  /* stands in for log(0): exp(x) == 0 <=> x < -745.13 */
#define LOG_ACC_BIT 28
#define LOG_STATE_BITS 14
#include "rx_walk2.cuh"
#include "rx_walk2c.cuh"
#include "rx_walk_exact.cuh"

// 24-bit row image of the energy matrix for the filter walkers: delta = u[k,l] - min_l u[k,l] as a float32 truncated to
// its top 24 bits (sign, 8 exponent, 15 mantissa bits), stored as a uint16 plane followed by a uint8 plane.  Relative
// precision 2^-15 per entry, so huge entries (a decoupled atom overlapping another one evaluated at lambda = 1) cost no
// precision where the decisions are made.  absmax_out[k] = max |u[k,:]| (inf for rows with non-finite values).
__global__ void k_mix_filter_build(const double *__restrict__ u, int K, unsigned char *__restrict__ filt, double *__restrict__ scale,
                                   double *__restrict__ absmax_out) {
    __shared__ double s_lo[8], s_am[8];
    const int k = blockIdx.x, t = threadIdx.x;
    double lo = INFINITY, am = 0.0;
    bool bad = false;
    for (int l = t; l < K; l += blockDim.x) {
        const double v = u[(size_t)k * K + l];
        if (!isfinite(v)) bad = true;
        lo = fmin(lo, v); am = fmax(am, fabs(v));
    }
    for (int o = 16; o > 0; o >>= 1) {
        lo = fmin(lo, __shfl_down_sync(0xffffffffu, lo, o));
        am = fmax(am, __shfl_down_sync(0xffffffffu, am, o));
    }
    const int anybad = __syncthreads_or(bad ? 1 : 0);
    if ((t & 31) == 0) { s_lo[t >> 5] = lo; s_am[t >> 5] = am; }
    __syncthreads();
    lo = s_lo[0]; am = s_am[0];
    for (int q = 1; q < (int)(blockDim.x >> 5); q++) { lo = fmin(lo, s_lo[q]); am = fmax(am, s_am[q]); }
    if (!isfinite(lo)) lo = 0.0;
    for (int l = t; l < K; l += blockDim.x) {
        const float f = (float)(u[(size_t)k * K + l] - lo);     // round to nearest f32; inf/NaN stay inf/NaN
        const unsigned bits = __float_as_uint(f) & 0xffffff00u;  // truncate to 24 bits (toward zero)
        ((unsigned short *)filt)[(size_t)k * K + l] = (unsigned short)(bits >> 16);
        filt[2 * (size_t)K * K + (size_t)k * K + l] = (unsigned char)((bits >> 8) & 0xffu);
    }
    if (t == 0) { scale[k] = fabs(lo); absmax_out[k] = anybad ? INFINITY : am; }
}

// Build the (symmetric) proposal / acceptance count matrices from entries [0, n) of a commit log (replicaexchange.py:339-349):
// the exact walker's dense log, or the filter walkers' sparse one (one word per record); bit 31 = an attempt is logged there.
__global__ void k_mix_count(const uint32_t *__restrict__ commit_log, long long n, int M, unsigned long long *__restrict__ nacc,
                            unsigned long long *__restrict__ nprop) {
    long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        const uint32_t e = commit_log[t];
        if (!(e >> 31)) continue;
        const uint32_t si = e & ((1u << LOG_STATE_BITS) - 1u), sj = (e >> LOG_STATE_BITS) & ((1u << LOG_STATE_BITS) - 1u);
        atomicAdd(&nprop[(size_t)si * M + sj], 1ull);
        atomicAdd(&nprop[(size_t)sj * M + si], 1ull);
        if ((e >> LOG_ACC_BIT) & 1u) {
            atomicAdd(&nacc[(size_t)si * M + sj], 1ull);
            atomicAdd(&nacc[(size_t)sj * M + si], 1ull);
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// Plain serial walker for any K (rejection sampling makes the slot structure state dependent).
// head counts WORDS here.  An attempt that would run out of words is rolled back.
// ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) k_mix_walk_serial(const uint32_t *__restrict__ words, long long nwords,
                                                        const double *__restrict__ u, int K, int M, int *perm_g,
                                                        unsigned long long *nacc, unsigned long long *nprop,
                                                        MixCtl *ctl) {
    extern __shared__ int s_perm[];
    const int lane = threadIdx.x;
    for (int q = lane; q < K; q += 32) s_perm[q] = perm_g[q];
    __syncwarp();
    if (lane == 0) {
        long long p = ctl->head, remaining = ctl->remaining;
        int nbits = 0;
        for (unsigned m = (unsigned)(K - 1); m; m >>= 1) nbits++;
        const uint32_t mask = nbits ? (0xffffffffu >> (32 - nbits)) : 0u;
        while (remaining > 0) {
            long long q = p;
            int i = 0, j = 0;
            bool ok = true;
            if (K > 1) {
                for (;;) { if (q >= nwords) { ok = false; break; } uint32_t r = words[q++] & mask; if ((int)r < K) { i = r; break; } }
                if (ok) for (;;) { if (q >= nwords) { ok = false; break; } uint32_t r = words[q++] & mask; if ((int)r < K) { j = r; break; } }
            }
            if (!ok) break;
            const int si = s_perm[i], sj = s_perm[j];
            const double logp = swap_logp(u[(size_t)i * M + sj], u[(size_t)j * M + si], u[(size_t)i * M + si],
                                          u[(size_t)j * M + sj]);
            bool acc = logp >= 0.0;
            if (!acc) {
                if (q + 2 > nwords) break;
                const double U = mt_double(words[q], words[q + 1]);
                q += 2;
                acc = U < rx_exp_cr(logp);
            }
            nprop[(size_t)si * M + sj] += 1;
            nprop[(size_t)sj * M + si] += 1;
            if (acc) {
                s_perm[i] = sj;
                s_perm[j] = si;
                nacc[(size_t)si * M + sj] += 1;
                nacc[(size_t)sj * M + si] += 1;
            }
            p = q;
            remaining--;
        }
        ctl->head = p;
        ctl->remaining = remaining;
        ctl->status = remaining > 0 ? 1 : 0;
    }
    __syncwarp();
    for (int q = lane; q < K; q += 32) perm_g[q] = s_perm[q];
}

// swap-neighbors (replicaexchange.py:366-406) on numpy's RandomState stream: offset = randint(2) is one
// masked word; each state pair (s, s+1) is attempted once; rand() (two words) only when log_p < 0.
__global__ void __launch_bounds__(32) k_mix_neighbors(const uint32_t *__restrict__ words, long long nwords,
                                                      const double *__restrict__ u, int K, int M, int *perm_g,
                                                      unsigned long long *nacc, unsigned long long *nprop,
                                                      MixCtl *ctl) {
    extern __shared__ int s_mem[];
    int *s_perm = s_mem, *s_inv = s_mem + K;
    const int lane = threadIdx.x;
    for (int q = lane; q < K; q += 32) { int s = perm_g[q]; s_perm[q] = s; if (s >= 0 && s < K) s_inv[s] = q; }
    __syncwarp();
    if (lane == 0) {
        long long p = 0;
        const int offset = (int)(words[p++] & 1u);
        for (int s = offset; s < K - 1; s += 2) {
            const int i = s_inv[s], j = s_inv[s + 1];
            const int si = s, sj = s + 1;
            const double logp = swap_logp(u[(size_t)i * M + sj], u[(size_t)j * M + si], u[(size_t)i * M + si],
                                          u[(size_t)j * M + sj]);
            bool acc = logp >= 0.0;
            if (!acc) {
                const double U = mt_double(words[p], words[p + 1]);
                p += 2;
                acc = U < rx_exp_cr(logp);
            }
            nprop[(size_t)si * M + sj] += 1;
            nprop[(size_t)sj * M + si] += 1;
            if (acc) {
                s_perm[i] = sj; s_perm[j] = si;
                s_inv[sj] = i; s_inv[si] = j;
                nacc[(size_t)si * M + sj] += 1;
                nacc[(size_t)sj * M + si] += 1;
            }
        }
        ctl->head = p;
        ctl->remaining = 0;
        ctl->status = 0;
    }
    __syncwarp();
    for (int q = lane; q < K; q += 32) perm_g[q] = s_perm[q];
}

// ------------------------------------------------------------------------------------------------------
// Host side: stream management
// ------------------------------------------------------------------------------------------------------
static int stream_reserve(rx_engine *h, MTStream &S, size_t cap) {
    if (cap <= S.cap) return RX_OK;
    DevBuf<uint32_t> a, b;
    RX_CHECK_CUDA(h, a.alloc(cap));
    RX_CHECK_CUDA(h, b.alloc(cap));
    if (S.avail) RX_CHECK_CUDA(h, cudaMemcpyAsync(a, S.d_words, S.avail * sizeof(uint32_t), cudaMemcpyDeviceToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaDeviceSynchronize());
    S.d_words = std::move(a); S.d_words_alt = std::move(b);
    S.cap = cap;
    return RX_OK;
}

// make at least `need` unconsumed words available
static int stream_fill(rx_engine *h, MTStream &S, size_t need, int *launches, cudaStream_t st) {
    if (S.avail >= need) return RX_OK;
    int rc = stream_reserve(h, S, need);
    if (rc) return rc;
    long long n = (long long)(need - S.avail);
    k_mt_generate<<<1, 256, 0, st>>>(S.d_window, S.d_words + S.avail, n);
    RX_CHECK_CUDA(h, cudaGetLastError());
    S.avail = need;
    (*launches)++;
    return RX_OK;
}

static int stream_consume(rx_engine *h, MTStream &S, size_t c, int *launches) {
    if (c > S.avail) RX_FAIL(h, RX_ERR_INVALID, "internal: consumed more words than available");
    size_t left = S.avail - c;
    if (left && c) {
        k_copy_words<<<(unsigned)((left + 1023) / 1024 > 1184 ? 1184 : (left + 1023) / 1024), 1024, 0, h->stream>>>(
            S.d_words + c, S.d_words_alt, (long long)left);
        RX_CHECK_CUDA(h, cudaGetLastError());
        std::swap(S.d_words, S.d_words_alt);
        (*launches)++;
    }
    S.avail = left;
    S.consumed += c;
    return RX_OK;
}

int rxi_mix_seed(rx_engine *h, int stream, uint32_t seed) {
    if (stream < 0 || stream > 1) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_seed: stream must be 0 (numba) or 1 (numpy)");
    MTStream &S = h->streams[stream];
    uint32_t mt[624];
    mt[0] = seed;  // init_genrand, numba/_random.c:59-73
    for (int i = 1; i < 624; i++) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
    if (!S.d_window) RX_CHECK_CUDA(h, S.d_window.alloc(624));
    RX_CHECK_CUDA(h, cudaMemcpy(S.d_window, mt, sizeof(mt), cudaMemcpyHostToDevice));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream_rng));
    if (stream == RX_STREAM_NUMBA) { h->prepared.valid = false; h->last_consumed = 0; }
    S.avail = 0;
    S.consumed = 0;
    S.seeded = true;
    return RX_OK;
}

int rxi_mix_skip(rx_engine *h, int stream, unsigned long long n) {
    if (stream < 0 || stream > 1) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_skip: stream must be 0 (numba) or 1 (numpy)");
    MTStream &S = h->streams[stream];
    if (!S.seeded) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_skip: seed the stream first");
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream_rng));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (stream == RX_STREAM_NUMBA) h->prepared.valid = false;
    // drop buffered words first, then advance the generator without storing
    const size_t c = (size_t)(n < S.avail ? n : S.avail);
    int launches = 0;
    int rc = stream_consume(h, S, c, &launches);
    if (rc) return rc;
    unsigned long long todo = n - c;
    while (todo > 0) {
        const long long chunk = todo > (1ull << 30) ? (1ll << 30) : (long long)todo;
        k_mt_generate<<<1, 256, 0, h->stream>>>(S.d_window, nullptr, chunk);
        RX_CHECK_CUDA(h, cudaGetLastError());
        todo -= (unsigned long long)chunk;
        S.consumed += (unsigned long long)chunk;
    }
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return RX_OK;
}

static inline bool is_pow2(int k) { return k >= 2 && (k & (k - 1)) == 0; }

// grid of the count kernels over n log entries: one thread per entry, at most 16 blocks per SM (grid-stride loop)
static inline unsigned count_blocks(const rx_engine *h, long long n) {
    const long long nb = (n + 255) / 256;
    return (unsigned)(nb < h->n_sm * 16 ? nb : h->n_sm * 16);
}

// number of candidates of the pass, behind the tile counts and their scan
static inline uint32_t *cand_total(const rx_engine *h) { return h->d_ctile + (h->ctile_cap / CAND_TILE + 4); }

// The speculative walkers are one latency-bound CTA each: they claim (almost) a whole SM's shared memory so that no other CTA --
// in particular the stream generator that runs concurrently on the side stream -- is scheduled onto the same SM and steals
// issue slots.  226 KB + the kernel's static shared memory + the generator's 8 KB exceed the SM's 228 KB.
#define WALK_SMEM (226 * 1024)

// The plan of a swap-all call: the records prepare_pass builds and the walkers of a pass.  A pass runs the bulk walker, if
// the plan has one, then the tail kernel, which continues from ctl.head:
//   coords      filter  K                              bulk              tail
//   slots       yes     power of two, <= 256           k_mix_walk2       k_mix_walk_pow2<true>
//   slots       no      power of two, <= 16384                           k_mix_walk_pow2<false>
//   candidates  yes     any other K in [3, 256]        k_mix_walk2c      k_mix_walk_serial
//   candidates  no      any other K in [3, ANY_MAX_K]  k_mix_walk_cand   k_mix_walk_serial
//   loop        no      every other K                                    k_mix_walk_serial
// RX_NO_FILTER=1 turns the filter off; RX_WALK_SERIAL=1 sends the K that would walk candidates to the plain loop.
static MixPlan mix_plan(int K) {
    MixPlan p = {MIX_LOOP, false, 1, (int)(K * sizeof(int))};
    if (is_pow2(K) && K <= (1 << LOG_STATE_BITS)) p = {MIX_SLOTS, false, 2, WALK_SMEM};
    else if (K >= 3 && K <= ANY_MAX_K && !getenv("RX_WALK_SERIAL")) p.coords = MIX_CANDS;
    // The f32 row-image filter wherever its walkers' shared memory fits (K <= 256; at K = 256 the 512 KB of f64 would not fit in
    // shared memory, and at smaller K the filter is still faster than f64 comparisons).  k_mix_walk2 / k_mix_walk2c hold ring,
    // replicas and image; k_mix_walk_pow2<true> ring, diag, rowabs, perm and image.
    const size_t smem_w2 = (size_t)W2_RING * 16 + (size_t)K * 8 + (size_t)((3 * K + 1) & ~1) * K;
    const size_t smem_f24 = (size_t)RING * 16 + (size_t)K * (2 * sizeof(double) + sizeof(int)) + (size_t)3 * K * K;
    p.filter = p.coords != MIX_LOOP && K <= 256 && smem_w2 <= 224 * 1024 && (p.coords == MIX_CANDS || smem_f24 <= 224 * 1024) &&
               !getenv("RX_NO_FILTER");
    return p;
}

static inline size_t pass_need(long long remaining, const MixPlan &p) {
    // words per pass (candidates: 16 bytes of records per word)
    const size_t chunk_words = p.coords == MIX_CANDS ? (size_t)1 << 25 : (size_t)1 << 26;
    size_t need = p.coords == MIX_SLOTS ? (size_t)(4 * remaining + 160) : (size_t)(8 * remaining + 512);
    if (need > chunk_words) need = chunk_words;
    if (need < 512) need = 512;
    return need;
}

// Top the stream up to what a pass over `remaining` attempts may consume and build the plan's records, on stream `st`.
// Both are state independent, so for the NEXT mixing call this runs on the side stream while the replicas are being
// propagated.
static int prepare_pass(rx_engine *h, MTStream &S, long long remaining, const MixPlan &p, int K, cudaStream_t st, int *launches) {
    static_assert(sizeof(SlotRec) == 16 && sizeof(SlotRec2) == 16 && sizeof(CandRec) == 16, "every record format fills one uint4");
    const bool cand = p.coords == MIX_CANDS;
    const size_t need = pass_need(remaining, p);
    int rc = stream_reserve(h, S, 2 * need + 1024);   // room for the words generated ahead while the walker runs
    if (rc) return rc;
    rc = stream_fill(h, S, need, launches, st);
    if (rc) return rc;
    if (p.coords != MIX_LOOP) {
        const long long nslots = cand ? (long long)S.avail : (long long)(S.avail / 2);   // records: per slot, or <= 1 per word
        if ((size_t)nslots > h->slots_cap) {
            // size for the largest stream the buffer can ever hold (2 * need + 1024 words), so that the slightly different
            // `avail` of every iteration never triggers another cudaFree/cudaMalloc (tens of ms each, device-synchronising)
            size_t want = cand ? S.cap : (S.cap + 1) / 2;
            if (want < (size_t)nslots) want = (size_t)nslots;
            DevBuf<uint4> slots;
            DevBuf<uint32_t> log, slotlog;
            RX_CHECK_CUDA(h, slots.alloc(want));
            RX_CHECK_CUDA(h, log.alloc(want));
            RX_CHECK_CUDA(h, slotlog.alloc(want));
            RX_CHECK_CUDA(h, cudaDeviceSynchronize());
            h->d_slots = std::move(slots); h->d_log = std::move(log); h->d_slotlog = std::move(slotlog);
            h->slots_cap = want;
        }
        if (cand && (!h->d_cpos || h->ctile_cap < h->slots_cap)) {
            DevBuf<uint32_t> cpos, ctile;
            RX_CHECK_CUDA(h, cpos.alloc(h->slots_cap + 8));
            RX_CHECK_CUDA(h, ctile.alloc(h->slots_cap / CAND_TILE + 8));
            RX_CHECK_CUDA(h, cudaDeviceSynchronize());
            h->d_cpos = std::move(cpos); h->d_ctile = std::move(ctile);
            h->ctile_cap = h->slots_cap;
        }
        if (cand) {
            // candidate coordinates (rx_walk2c.cuh): flag + count per tile, scan, scatter, one record per candidate index
            int nbits = 0;
            for (unsigned m = (unsigned)(K - 1); m; m >>= 1) nbits++;
            const uint32_t mask = 0xffffffffu >> (32 - nbits);
            const int ntiles = (int)((nslots + CAND_TILE - 1) / CAND_TILE);
            const unsigned nblk = (unsigned)((nslots + 255) / 256);
            k_cand_count<<<ntiles, 256, 0, st>>>(S.d_words, nslots, K, mask, h->d_ctile);
            k_cand_scan<<<1, 1024, 0, st>>>(h->d_ctile, ntiles, cand_total(h));
            k_cand_scatter<<<ntiles, 256, 0, st>>>(S.d_words, nslots, K, mask, h->d_ctile, h->d_cpos);
            if (p.filter)
                k_cand_records<false><<<nblk, 256, 0, st>>>(S.d_words, h->d_cpos, cand_total(h), mask, (SlotRec2 *)h->d_slots.get());
            else
                k_cand_records<true><<<nblk, 256, 0, st>>>(S.d_words, h->d_cpos, cand_total(h), mask, (CandRec *)h->d_slots.get());
            *launches += 3;
        } else if (p.filter)
            k_slots_build<true><<<(unsigned)((nslots + 255) / 256), 256, 0, st>>>(S.d_words, nslots, (uint32_t)(K - 1), (SlotRec2 *)h->d_slots.get());
        else
            k_slots_build<false><<<(unsigned)((nslots + 255) / 256), 256, 0, st>>>(S.d_words, nslots, (uint32_t)(K - 1), (SlotRec *)h->d_slots.get());
        RX_CHECK_CUDA(h, cudaGetLastError());
        (*launches)++;
    }
    h->prepared = {false, p, S.avail};
    return RX_OK;
}

int rxi_mix_swap_all(rx_engine *h, long long nswap, int *launches) {
    MTStream &S = h->streams[RX_STREAM_NUMBA];
    if (!S.seeded) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_swap_all: the numba MT19937 stream has not been seeded (rx_mix_seed)");
    const int K = h->cfg.n_replicas, M = h->cfg.n_states;
    if (K != M) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_swap_all: requires n_replicas == n_states");
    const size_t mm = (size_t)M * M * sizeof(unsigned long long);
    RX_CHECK_CUDA(h, cudaMemsetAsync(h->d_nacc, 0, mm, h->stream));
    RX_CHECK_CUDA(h, cudaMemsetAsync(h->d_nprop, 0, mm, h->stream));
    if (nswap <= 0) return RX_OK;
    if (K == 1) {  // randint(1) draws nothing, log_p == 0: every attempt is an accepted no-op
        unsigned long long two_n = 2ull * (unsigned long long)nswap;
        RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_nacc, &two_n, 8, cudaMemcpyHostToDevice, h->stream));
        RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_nprop, &two_n, 8, cudaMemcpyHostToDevice, h->stream));
        RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
        return RX_OK;
    }
    const MixPlan p = mix_plan(K);
    int logK = 0;
    while ((1 << logK) < K) logK++;
    // the plan's walkers and their dynamic shared memory
    const void *bulk = !p.filter ? (p.coords == MIX_CANDS ? (const void *)k_mix_walk_cand : nullptr)
                                 : (p.coords == MIX_SLOTS ? (const void *)k_mix_walk2 : (const void *)k_mix_walk2c);
    const auto walk_pow2 = p.filter ? k_mix_walk_pow2<true> : k_mix_walk_pow2<false>;
    const void *tail = p.coords == MIX_SLOTS ? (const void *)walk_pow2 : (const void *)k_mix_walk_serial;
    if (bulk) RX_CHECK_CUDA(h, cudaFuncSetAttribute(bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, WALK_SMEM));
    if (p.smem_tail > 48 * 1024) RX_CHECK_CUDA(h, cudaFuncSetAttribute(tail, cudaFuncAttributeMaxDynamicSharedMemorySize, p.smem_tail));
    if (p.filter) {
        if (!h->d_filt) {
            DevBuf<unsigned char> filt;
            DevBuf<double> scale;
            RX_CHECK_CUDA(h, filt.alloc((size_t)3 * K * K + 16));
            RX_CHECK_CUDA(h, scale.alloc(2 * (size_t)K));
            h->d_filt = std::move(filt); h->d_filt_scale = std::move(scale);
        }
        // row image + |row minimum| for the per-lane error bound; non-finite or astronomically large entries only send the
        // lanes that touch them to the exact path (no host round trip, no global fallback)
        k_mix_filter_build<<<K, 256, 0, h->stream>>>(h->d_u, K, h->d_filt, h->d_filt_scale, h->d_filt_scale + K);
        RX_CHECK_CUDA(h, cudaGetLastError());
        (*launches)++;
    }
    long long remaining = nswap;
    h->mix_stats[0] = h->mix_stats[1] = h->mix_stats[2] = h->mix_stats[4] = h->mix_stats[5] = 0;
    const uint64_t consumed0 = S.consumed;
    const size_t chunk_words = (size_t)1 << 26;
    while (remaining > 0) {
        const size_t need = pass_need(remaining, p);
        int rc;
        if (h->prepared.valid && h->prepared.plan == p && S.avail >= need && h->prepared.avail == S.avail) {
            // produced on the side stream while the replicas were propagating
            RX_CHECK_CUDA(h, cudaStreamWaitEvent(h->stream, h->ev_prepared, 0));
            float ms = 0;
            const double tw0 = rx_wall_us();
            if (cudaEventSynchronize(h->ev[7]) == cudaSuccess && cudaEventElapsedTime(&ms, h->ev[6], h->ev[7]) == cudaSuccess)
                h->phase_ms[3] += ms;
            h->mix_stats[5] += (long long)(rx_wall_us() - tw0);
        } else {
            if (h->prepared.valid) RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream_rng));
            rc = prepare_pass(h, S, remaining, p, K, h->stream, launches);
            if (rc) return rc;
        }
        h->prepared.valid = false;
        MixCtl ctl = {0, remaining, 0, 0, 0, 0, 0};
        RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_ctl, &ctl, sizeof(ctl), cudaMemcpyHostToDevice, h->stream));
        const size_t nrec = p.coords == MIX_SLOTS ? S.avail / 2 : S.avail;   // records: per slot, or <= 1 per word
        // Passes over slots: while the walkers run (they only read words [0, avail)), generate on the side stream about as many
        // words as the previous call consumed; they are appended behind the valid region and adopted afterwards.
        size_t ahead = 0;
        if (p.coords == MIX_SLOTS && !getenv("RX_NO_ASYNC_RNG") && h->last_consumed > 0 && S.avail + h->last_consumed <= S.cap) {
            ahead = h->last_consumed;
            k_mt_generate<<<1, 256, 0, h->stream_rng>>>(S.d_window, S.d_words + S.avail, (long long)ahead);
            RX_CHECK_CUDA(h, cudaGetLastError());
            RX_CHECK_CUDA(h, cudaEventRecord(h->ev_prepared, h->stream_rng));
            *launches += 1;
        }
        // walker_ms times the speculative walkers of a pass (the bulk walker, and k_mix_walk_pow2 over slots), never the plain loop
        const bool timed = p.coords != MIX_LOOP;
        if (timed) RX_CHECK_CUDA(h, cudaEventRecord(h->ev_walk[0], h->stream));
        if (p.filter) {
            // the filter walker logs the attempts it commits sparsely, one word per record (zero = no attempt started there),
            // and reports the extent of that log in ctl.aux
            RX_CHECK_CUDA(h, cudaMemsetAsync(h->d_slotlog, 0, nrec * sizeof(uint32_t), h->stream));
            if (p.coords == MIX_SLOTS)
                k_mix_walk2<<<1, W2_THREADS, WALK_SMEM, h->stream>>>((const SlotRec2 *)h->d_slots.get(), S.d_words, (unsigned)nrec, h->d_u, K,
                                                                   logK, h->d_perm, h->d_slotlog, h->d_filt, h->d_filt_scale, h->d_ctl);
            else
                k_mix_walk2c<<<1, W2_THREADS, WALK_SMEM, h->stream>>>((const SlotRec2 *)h->d_slots.get(), S.d_words, h->d_cpos, cand_total(h),
                                                                    h->d_u, K, h->d_perm, h->d_slotlog, h->d_filt, h->d_filt_scale,
                                                                    h->d_ctl);
        } else if (p.coords == MIX_CANDS)
            k_mix_walk_cand<<<1, 64, WALK_SMEM, h->stream>>>((const CandRec *)h->d_slots.get(), S.d_words, h->d_cpos, cand_total(h), h->d_u, K,
                                                               h->d_perm, h->d_log, h->d_ctl);
        if (bulk) {
            RX_CHECK_CUDA(h, cudaGetLastError());
            *launches += 1;
        }
        // the pass's tail continues from ctl.head
        if (p.coords == MIX_SLOTS)
            walk_pow2<<<1, 64, p.smem_tail, h->stream>>>((const SlotRec *)h->d_slots.get(), S.d_words, (unsigned)nrec, h->d_u, K, logK, h->d_perm,
                                                         h->d_log, p.filter ? h->d_filt.get() : nullptr, p.filter ? h->d_filt_scale.get() : nullptr, h->d_ctl);
        if (timed) RX_CHECK_CUDA(h, cudaEventRecord(h->ev_walk[1], h->stream));
        if (p.coords != MIX_SLOTS)
            k_mix_walk_serial<<<1, 32, p.smem_tail, h->stream>>>(S.d_words, (long long)S.avail, h->d_u, K, M, h->d_perm, h->d_nacc,
                                                                 h->d_nprop, h->d_ctl);
        RX_CHECK_CUDA(h, cudaGetLastError());
        *launches += 1;
        RX_CHECK_CUDA(h, cudaMemcpyAsync(&ctl, h->d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost, h->stream));
        RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
        float wms = 0;
        if (timed && cudaEventElapsedTime(&wms, h->ev_walk[0], h->ev_walk[1]) == cudaSuccess) h->mix_stats[4] += (long long)(wms * 1e3f);
        const size_t consumed_words = (size_t)ctl.head * p.head_unit;
        if (ahead) {   // adopt the words generated during the walk
            RX_CHECK_CUDA(h, cudaStreamWaitEvent(h->stream, h->ev_prepared, 0));
            S.avail += ahead;
        }
        // count matrices from the commit logs (k_mix_walk_serial counts as it goes)
        if (ctl.aux > 0) {   // the filter walker's sparse log
            k_mix_count<<<count_blocks(h, ctl.aux), 256, 0, h->stream>>>(h->d_slotlog, ctl.aux, M, h->d_nacc, h->d_nprop);
            RX_CHECK_CUDA(h, cudaGetLastError());
            *launches += 1;
        }
        if (ctl.log_count > 0) {   // the dense log of k_mix_walk_pow2 / k_mix_walk_cand
            k_mix_count<<<count_blocks(h, ctl.log_count), 256, 0, h->stream>>>(h->d_log, ctl.log_count, M, h->d_nacc, h->d_nprop);
            RX_CHECK_CUDA(h, cudaGetLastError());
            *launches += 1;
        }
        if (ctl.remaining == remaining && consumed_words == 0 && need >= chunk_words)
            RX_FAIL(h, RX_ERR_INVALID, "internal: mixing made no progress");
        remaining = ctl.remaining;
        h->mix_stats[0] += ctl.rounds;
        h->mix_stats[1] += ctl.slow_exp;
        h->mix_stats[2] += 1;
        rc = stream_consume(h, S, consumed_words, launches);
        if (rc) return rc;
    }
    h->mix_stats[3] = (long long)(S.consumed - consumed0);
    h->last_consumed = (size_t)(S.consumed - consumed0);
    if (!getenv("RX_NO_ASYNC_RNG")) {
        // overlap the next call's stream generation + slot records with whatever runs next on the main stream
        RX_CHECK_CUDA(h, cudaEventRecord(h->ev_consumed, h->stream));
        RX_CHECK_CUDA(h, cudaStreamWaitEvent(h->stream_rng, h->ev_consumed, 0));
        RX_CHECK_CUDA(h, cudaEventRecord(h->ev[6], h->stream_rng));
        int l2 = 0;
        int rc2 = prepare_pass(h, S, nswap, p, K, h->stream_rng, &l2);
        if (rc2) return rc2;
        RX_CHECK_CUDA(h, cudaEventRecord(h->ev[7], h->stream_rng));
        RX_CHECK_CUDA(h, cudaEventRecord(h->ev_prepared, h->stream_rng));
        h->phase_launches[3] += l2;
        h->prepared.valid = true;
    }
    return RX_OK;
}

int rxi_mix_swap_neighbors(rx_engine *h, int *launches) {
    MTStream &S = h->streams[RX_STREAM_NUMPY];
    if (!S.seeded) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_swap_neighbors: the numpy MT19937 stream has not been seeded (rx_mix_seed)");
    const int K = h->cfg.n_replicas, M = h->cfg.n_states;
    if (K != M) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_swap_neighbors: requires n_replicas == n_states");
    const size_t mm = (size_t)M * M * sizeof(unsigned long long);
    RX_CHECK_CUDA(h, cudaMemsetAsync(h->d_nacc, 0, mm, h->stream));
    RX_CHECK_CUDA(h, cudaMemsetAsync(h->d_nprop, 0, mm, h->stream));
    int rc = stream_fill(h, S, (size_t)K + 64, launches, h->stream);
    if (rc) return rc;
    const size_t smem = 2 * (size_t)K * sizeof(int);
    if (smem > 48 * 1024)
        RX_CHECK_CUDA(h, cudaFuncSetAttribute(k_mix_neighbors, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MixCtl ctl = {0, 0, 0, 0, 0, 0};
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_ctl, &ctl, sizeof(ctl), cudaMemcpyHostToDevice, h->stream));
    k_mix_neighbors<<<1, 32, smem, h->stream>>>(S.d_words, (long long)S.avail, h->d_u, K, M, h->d_perm, h->d_nacc, h->d_nprop,
                                              h->d_ctl);
    RX_CHECK_CUDA(h, cudaGetLastError());
    (*launches)++;
    RX_CHECK_CUDA(h, cudaMemcpyAsync(&ctl, h->d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost, h->stream));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return stream_consume(h, S, (size_t)ctl.head, launches);
}

#include "rx_sams.cuh"
