// rx_mbar.cu -- the two passes of an MBAR solve over a device-resident reduced-potential matrix (DESIGN §4.7).
//
// Shirts & Chodera 2008: with c_k = log N_k + f_k, the density of sample n is log D_n = logsumexp_k (c_k - u_kn) and its
// weight in state i is W_in = exp(f_i - u_in - log D_n).  At creation k_mbar_shift subtracts m_n = min over the sampled
// states of u_kn from every sample: W is unchanged, and exp's argument no longer carries the rounding of |u| ~ 1e5 kT.
// Pass 1 (k_mbar_logden) writes log D_n of the shifted u; pass 2 reduces W over the samples: k_mbar_rowsum gives
// log sum_n W_in (a log-sum-exp, so it neither underflows nor overflows at any energy scale) and sum_n log D_n,
// k_mbar_gram gives sum_n W_in W_jn.  Every reduction is cut into chunks of samples whose number depends on K and N only;
// a chunk is summed by one block in a fixed order and the chunks are then combined by a fixed pairwise tree
// (k_mbar_tree, k_mbar_tree_rows), so results do not depend on the grid.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <string>
#include <vector>
#include "rx_internal.cuh"

namespace {

constexpr int GT = 64;            // Gram output tile edge (states)
constexpr int GS = 16;            // samples per shared-memory step of the Gram tile
constexpr int GTHREADS = 256;     // 16 x 16 threads, 4 x 4 outputs each
constexpr int RTHREADS = 256;     // k_mbar_rowsum block
constexpr int ROW_CHUNK = 8192;   // samples per k_mbar_rowsum chunk
constexpr int GRAM_WORK = 2048;   // k_mbar_gram aims at this many (tile pair, chunk) work items

// u_kn row i, sample n -> W_in; 0 outside the matrix
__device__ __forceinline__ double weight(const double *__restrict__ u, size_t N, int K, int i, long long n,
                                         const double *__restrict__ f, const double *__restrict__ logD) {
    if (i >= K || n >= (long long)N) return 0.0;
    return exp(f[i] - u[(size_t)i * N + n] - logD[n]);
}

// Pass 1: one thread per sample, a running log-sum-exp over the states in index order.  States with c_k = -inf (no
// samples) add nothing and never become the running maximum.
__global__ void k_mbar_logden(const double *__restrict__ u, size_t N, int K, const double *__restrict__ c,
                              double *__restrict__ logD) {
    for (long long n = blockIdx.x * (long long)blockDim.x + threadIdx.x; n < (long long)N;
         n += (long long)gridDim.x * blockDim.x) {
        double m = -INFINITY, s = 0.0;
        for (int k = 0; k < K; ++k) {
            const double ck = c[k];
            if (ck == -INFINITY) continue;
            const double v = ck - u[(size_t)k * N + n];
            if (v > m) { s = s * exp(m - v) + 1.0; m = v; }
            else s += exp(v - m);
        }
        logD[n] = m + log(s);
    }
}

// (m, s) += (m2, s2) for running log-sum-exps m + log s; (-inf, 0) is the empty sum.  One exp per call.
__device__ __forceinline__ void lse_add(double &m, double &s, double m2, double s2) {
    if (m2 > m) { s = s * exp(m - m2) + s2; m = m2; }   // s = 0 while m = -inf, so exp(-inf) = 0 adds nothing
    else if (m2 != -INFINITY) s += s2 * exp(m2 - m);
}

// sum over a block of RTHREADS in a fixed order
__device__ double block_sum(double v, double *sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = RTHREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}

// (m, s) log-sum-exp over a block of RTHREADS in the same fixed order; the result is in (m, s) of thread 0
__device__ void block_lse(double &m, double &s, double *shm, double *shs) {
    shm[threadIdx.x] = m;
    shs[threadIdx.x] = s;
    __syncthreads();
    for (int o = RTHREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            double a = shm[threadIdx.x], b = shs[threadIdx.x];
            lse_add(a, b, shm[threadIdx.x + o], shs[threadIdx.x + o]);
            shm[threadIdx.x] = a;
            shs[threadIdx.x] = b;
        }
        __syncthreads();
    }
    m = shm[0];
    s = shs[0];
    __syncthreads();
}

// Pass 2a: work item (row r, chunk c) -> the record pair part[c * 2 (K + 1) + 2 r ..] = (m, s) with
// m + log s = log sum over the chunk's samples of W_rn (r < K), or (sum of log D_n - m_n, 0) for r = K.  Each thread
// runs over a strided subsequence of the chunk in order, then the block combines the threads.
__global__ void k_mbar_rowsum(const double *__restrict__ u, size_t N, int K, const double *__restrict__ f,
                              const double *__restrict__ logD, const double *__restrict__ shift, int n_chunks,
                              double *__restrict__ part) {
    __shared__ double shm[RTHREADS], shs[RTHREADS];
    const long long items = (long long)(K + 1) * n_chunks;
    for (long long w = blockIdx.x; w < items; w += gridDim.x) {
        const int r = (int)(w % (K + 1)), c = (int)(w / (K + 1));
        const long long n0 = (long long)c * ROW_CHUNK, n1 = min(n0 + ROW_CHUNK, (long long)N);
        double m, s;
        if (r < K) {
            m = -INFINITY;
            s = 0.0;
            const double fr = f[r];
            for (long long n = n0 + threadIdx.x; n < n1; n += RTHREADS) {
                const double v = fr - u[(size_t)r * N + n] - logD[n];
                if (v > m) { s = s * exp(m - v) + 1.0; m = v; }
                else s += exp(v - m);
            }
            block_lse(m, s, shm, shs);
        } else {
            m = 0.0;
            for (long long n = n0 + threadIdx.x; n < n1; n += RTHREADS) m += logD[n] - shift[n];
            m = block_sum(m, shm);
            s = 0.0;
        }
        if (threadIdx.x == 0) {
            part[((size_t)c * (K + 1) + r) * 2] = m;
            part[((size_t)c * (K + 1) + r) * 2 + 1] = s;
        }
    }
}

// Pass 2b: work item (tile pair p = (I, J) with I <= J, chunk c) -> the 64 x 64 block G[I-tile][J-tile] summed over the
// chunk's samples, at part[(c * n_pairs + p) * 4096].  Per step of GS samples the block stages W of both row tiles,
// transposed (sample-major), in shared memory; thread (tx, ty) owns rows ty + 16 a and columns tx + 16 b (a, b < 4), so
// a warp reads its J-row operands from consecutive addresses and its I-row operands as broadcasts.
__global__ void __launch_bounds__(GTHREADS) k_mbar_gram(const double *__restrict__ u, size_t N, int K,
                                                        const double *__restrict__ f, const double *__restrict__ logD,
                                                        int n_tiles, int n_pairs, int n_chunks, long long chunk,
                                                        double *__restrict__ part) {
    __shared__ double sA[GS][GT + 1], sB[GS][GT + 1];
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    const long long items = (long long)n_pairs * n_chunks;
    for (long long w = blockIdx.x; w < items; w += gridDim.x) {
        int p = (int)(w % n_pairs), I = 0;
        const int c = (int)(w / n_pairs);
        while (p >= n_tiles - I) { p -= n_tiles - I; ++I; }   // p-th pair of the upper triangle, row-major
        const int J = I + p;
        const long long n0 = c * chunk, n1 = min(n0 + chunk, (long long)N);
        double acc[4][4] = {};
        for (long long s0 = n0; s0 < n1; s0 += GS) {
            // 64 rows x GS samples per tile: thread t stages row t / 4, samples 4 (t % 4) .. + 3
            const int row = threadIdx.x / 4, col = 4 * (threadIdx.x % 4);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const long long n = s0 + col + q;
                const bool in = n < n1;
                sA[col + q][row] = in ? weight(u, N, K, I * GT + row, n, f, logD) : 0.0;
                if (I != J) sB[col + q][row] = in ? weight(u, N, K, J * GT + row, n, f, logD) : 0.0;
            }
            __syncthreads();
            const double(*B)[GT + 1] = I == J ? sA : sB;
#pragma unroll
            for (int s = 0; s < GS; ++s) {
                double a[4], b[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) { a[q] = sA[s][ty + 16 * q]; b[q] = B[s][tx + 16 * q]; }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
            }
            __syncthreads();
        }
        double *out = part + ((size_t)c * n_pairs + (I * n_tiles - I * (I - 1) / 2 + (J - I))) * (GT * GT);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) out[(ty + 16 * i) * GT + tx + 16 * j] = acc[i][j];
    }
}

// u_kn from the engine's energy history (rx_mbar_create_from_history): u[i][r n_sel + j] = hist[iter[j]][r][cols[i]].  A
// block transposes a tile of TT samples (one replica, TT consecutive selected iterations) x TT rows of u_kn through shared
// memory: a warp reads TT states of one history row and writes TT consecutive samples of one u_kn row.  Any non-finite
// element sets *bad.
constexpr int TT = 32, TROWS = 8;
__global__ void __launch_bounds__(TT * TROWS) k_mbar_gather(const double *__restrict__ hist, int R, int W,
                                                            const long long *__restrict__ iter, int n_sel, int j_tiles,
                                                            const int *__restrict__ cols, int K, double *__restrict__ u,
                                                            int *__restrict__ bad) {
    __shared__ double t[TT][TT + 1];
    const int r = blockIdx.x / j_tiles, j0 = (blockIdx.x % j_tiles) * TT, i0 = blockIdx.y * TT;
    const size_t N = (size_t)R * n_sel;
    bool finite = true;
    const int i = i0 + threadIdx.x;
    const int col = i < K ? cols[i] : 0;
    for (int s = threadIdx.y; s < TT; s += TROWS) {
        const int j = j0 + s;
        if (i < K && j < n_sel) {
            const double v = hist[((size_t)iter[j] * R + r) * W + col];
            finite &= isfinite(v);
            t[s][threadIdx.x] = v;
        }
    }
    __syncthreads();
    const int j = j0 + threadIdx.x;
    for (int s = threadIdx.y; s < TT; s += TROWS)
        if (i0 + s < K && j < n_sel) u[(size_t)(i0 + s) * N + (size_t)r * n_sel + j] = t[threadIdx.x][s];
    if (!finite) atomicExch(bad, 1);
}

// One level of the fixed pairwise tree over chunk records of len doubles: rec[c] += rec[c + half] for c < n - half.
__global__ void k_mbar_tree(double *__restrict__ rec, size_t len, int n, int half) {
    const size_t total = (size_t)(n - half) * len;
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x)
        rec[e] += rec[e + (size_t)half * len];
}

// The same tree over k_mbar_rowsum's records of K + 1 pairs: pair r < K of rec[c] is log-sum-exp combined with that of
// rec[c + half], pair K is added.
__global__ void k_mbar_tree_rows(double *__restrict__ rec, int K, int n, int half) {
    const size_t total = (size_t)(n - half) * (K + 1), len = 2 * (size_t)(K + 1);
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const size_t c = e / (K + 1), r = e % (K + 1);
        double *a = rec + c * len + 2 * r;
        const double *b = a + (size_t)half * len;
        if (r < (size_t)K) lse_add(a[0], a[1], b[0], b[1]);
        else a[0] += b[0];
    }
}

// One thread per sample: m_n = min over the sampled states (c_k = log N_k > -inf) of u_kn, then u_kn -= m_n for every
// state, sampled or not.  MBAR's f and W are unchanged by any per-sample shift; this one makes the sampled states' u
// at least 0 and 0 for one of them, so log D_n and exp's arguments are of the order of the spread across states
// instead of |u|.
__global__ void k_mbar_shift(double *__restrict__ u, size_t N, int K, const double *__restrict__ c,
                             double *__restrict__ shift) {
    for (long long n = blockIdx.x * (long long)blockDim.x + threadIdx.x; n < (long long)N;
         n += (long long)gridDim.x * blockDim.x) {
        double m = INFINITY;
        for (int k = 0; k < K; ++k)
            if (c[k] != -INFINITY) m = fmin(m, u[(size_t)k * N + n]);
        for (int k = 0; k < K; ++k) u[(size_t)k * N + n] -= m;
        shift[n] = m;
    }
}

}  // namespace

struct rx_mbar {
    int K = 0;
    size_t N = 0;
    int device = 0;              // the current device at rx_mbar_create
    int n_sm = 0;
    int max_blocks = 0;          // rx_mbar_set_max_blocks (0: from the device)
    std::vector<double> logN;    // log N_k, -inf for N_k = 0
    std::vector<double> Nk;
    int row_chunks = 0;          // k_mbar_rowsum chunks
    int n_tiles = 0, n_pairs = 0, gram_chunks = 0;
    long long gram_chunk = 0;    // samples per k_mbar_gram chunk (a multiple of GS)
    DevBuf<double> d_u, d_logD, d_shift, d_c, d_f, d_rows, d_gram;
    std::vector<double> h_rows, h_gram;   // h_rows: (m, s) of log sum_n W_in for i < K, then (sum_n log D_n, 0)
    std::vector<double> log_wsum;         // log sum_n W_in of the last run
    cudaStream_t stream = nullptr;
    std::string err;
    ~rx_mbar() { if (stream) cudaStreamDestroy(stream); }
};

namespace {

thread_local std::string g_mbar_create_error;

int blocks_for(const rx_mbar *h, long long items, int per_sm) {
    long long b = h->max_blocks > 0 ? h->max_blocks : (long long)h->n_sm * per_sm;
    return (int)std::max(1LL, std::min(items, b));
}

// sums n_chunks records of len doubles in place into rec[0]
int tree(rx_mbar *h, double *rec, size_t len, int n) {
    while (n > 1) {
        const int half = (n + 1) / 2;
        const long long work = (long long)(n - half) * (long long)len;
        k_mbar_tree<<<blocks_for(h, (work + 255) / 256, 16), 256, 0, h->stream>>>(rec, len, n, half);
        RX_CHECK_CUDA(h, cudaGetLastError());
        n = half;
    }
    return RX_OK;
}

// The K + 1 row records: (m, s) pairs of k_mbar_rowsum, combined into rec[0] by the tree.
int tree_rows(rx_mbar *h, double *rec, int n) {
    const int K = h->K;
    while (n > 1) {
        const int half = (n + 1) / 2;
        const long long work = (long long)(n - half) * (K + 1);
        k_mbar_tree_rows<<<blocks_for(h, (work + 255) / 256, 16), 256, 0, h->stream>>>(rec, K, n, half);
        RX_CHECK_CUDA(h, cudaGetLastError());
        n = half;
    }
    return RX_OK;
}

// log D at f, then log sum_n W_in and sum_n log D_n (h_rows, log_wsum) and, when gram, sum_n W_in W_jn (h_gram, upper tile pairs)
int run(rx_mbar *h, const double *f, bool gram) {
    const int K = h->K;
    RX_CHECK_CUDA(h, cudaSetDevice(h->device));
    std::vector<double> c(K);
    for (int k = 0; k < K; ++k) {
        if (!isfinite(f[k])) RX_FAIL(h, RX_ERR_INVALID, "f_k must be finite");
        c[k] = h->logN[k] + f[k];
    }
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_c, c.data(), K * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->d_f, f, K * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    k_mbar_logden<<<blocks_for(h, ((long long)h->N + 255) / 256, 16), 256, 0, h->stream>>>(h->d_u, h->N, K, h->d_c,
                                                                                              h->d_logD);
    RX_CHECK_CUDA(h, cudaGetLastError());
    k_mbar_rowsum<<<blocks_for(h, (long long)(K + 1) * h->row_chunks, 8), RTHREADS, 0, h->stream>>>(
        h->d_u, h->N, K, h->d_f, h->d_logD, h->d_shift, h->row_chunks, h->d_rows);
    RX_CHECK_CUDA(h, cudaGetLastError());
    int rc = tree_rows(h, h->d_rows, h->row_chunks);
    if (rc) return rc;
    RX_CHECK_CUDA(h, cudaMemcpyAsync(h->h_rows.data(), h->d_rows, 2 * (K + 1) * sizeof(double),
                                     cudaMemcpyDeviceToHost, h->stream));
    if (gram) {
        k_mbar_gram<<<blocks_for(h, (long long)h->n_pairs * h->gram_chunks, 8), GTHREADS, 0, h->stream>>>(
            h->d_u, h->N, K, h->d_f, h->d_logD, h->n_tiles, h->n_pairs, h->gram_chunks, h->gram_chunk, h->d_gram);
        RX_CHECK_CUDA(h, cudaGetLastError());
        rc = tree(h, h->d_gram, (size_t)h->n_pairs * GT * GT, h->gram_chunks);
        if (rc) return rc;
        RX_CHECK_CUDA(h, cudaMemcpyAsync(h->h_gram.data(), h->d_gram, h->h_gram.size() * sizeof(double),
                                         cudaMemcpyDeviceToHost, h->stream));
    }
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    // every row has N >= 1 samples, so m is finite and s >= 1
    for (int i = 0; i < K; ++i) h->log_wsum[i] = h->h_rows[2 * i] + log(h->h_rows[2 * i + 1]);
    return RX_OK;
}

// the full K x K Gram matrix from the upper tile pairs of h_gram
void unpack_gram(const rx_mbar *h, double *G) {
    const int K = h->K, T = h->n_tiles;
    for (int i = 0; i < K; ++i)
        for (int j = i; j < K; ++j) {
            const int I = i / GT, J = j / GT;
            const size_t p = (size_t)I * T - (size_t)I * (I - 1) / 2 + (J - I);
            const double v = h->h_gram[p * GT * GT + (i % GT) * GT + (j % GT)];
            G[(size_t)i * K + j] = v;
            G[(size_t)j * K + i] = v;
        }
}

}  // namespace

extern "C" const char *rx_mbar_last_error(const rx_mbar *h) { return h ? h->err.c_str() : g_mbar_create_error.c_str(); }

#define MBAR_CREATE_FAIL(code, msg) do { g_mbar_create_error = (msg); return (code); } while (0)

// A handle with every device buffer allocated on the current device; u_kn still to be filled.  `extra` bytes of the
// caller's are part of the free-memory check.
static int mbar_alloc(int32_t K, int64_t N, const int64_t *N_k, size_t extra, std::unique_ptr<rx_mbar> &out) {
    long long total = 0;
    for (int k = 0; k < K; ++k) {
        if (N_k[k] < 0) MBAR_CREATE_FAIL(RX_ERR_INVALID, "rx_mbar_create: N_k must be non-negative");
        total += N_k[k];
    }
    if (total != N) MBAR_CREATE_FAIL(RX_ERR_INVALID, "rx_mbar_create: sum of N_k must equal N");
    auto h = std::make_unique<rx_mbar>();
    h->K = K;
    h->N = (size_t)N;
    h->row_chunks = (int)((N + ROW_CHUNK - 1) / ROW_CHUNK);
    h->n_tiles = (K + GT - 1) / GT;
    h->n_pairs = h->n_tiles * (h->n_tiles + 1) / 2;
    // chunks of the Gram pass: about GRAM_WORK work items, at least 2 * GS samples each
    long long want = std::max(1, GRAM_WORK / h->n_pairs);
    want = std::min(want, std::max(1LL, (long long)N / (2 * GS)));
    h->gram_chunk = ((N + want - 1) / want + GS - 1) / GS * GS;
    h->gram_chunks = (int)((N + h->gram_chunk - 1) / h->gram_chunk);
    const size_t bytes = (size_t)K * N * sizeof(double) + 2 * (size_t)N * sizeof(double) +
                         (size_t)h->row_chunks * 2 * (K + 1) * sizeof(double) +
                         (size_t)h->gram_chunks * h->n_pairs * GT * GT * sizeof(double) + extra;
    if (cudaGetDevice(&h->device) != cudaSuccess) MBAR_CREATE_FAIL(RX_ERR_CUDA, "rx_mbar_create: no CUDA device");
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) MBAR_CREATE_FAIL(RX_ERR_CUDA, "rx_mbar_create: cudaMemGetInfo failed");
    // the size is checked before u_kn is read
    if (bytes > free_b)
        MBAR_CREATE_FAIL(RX_ERR_UNSUPPORTED, "rx_mbar_create: u_kn and its reduction buffers need " + std::to_string(bytes) +
                                                 " bytes, the device has " + std::to_string(free_b) + " free");
    if (cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, h->device) != cudaSuccess)
        MBAR_CREATE_FAIL(RX_ERR_CUDA, "rx_mbar_create: cudaDeviceGetAttribute failed");
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess)
        MBAR_CREATE_FAIL(RX_ERR_CUDA, "rx_mbar_create: cudaStreamCreate failed");
    cudaError_t e = h->d_u.alloc((size_t)K * N);
    if (e == cudaSuccess) e = h->d_logD.alloc(N);
    if (e == cudaSuccess) e = h->d_shift.alloc(N);
    if (e == cudaSuccess) e = h->d_c.alloc(K);
    if (e == cudaSuccess) e = h->d_f.alloc(K);
    if (e == cudaSuccess) e = h->d_rows.alloc((size_t)h->row_chunks * 2 * (K + 1));
    if (e == cudaSuccess) e = h->d_gram.alloc((size_t)h->gram_chunks * h->n_pairs * GT * GT);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        MBAR_CREATE_FAIL(RX_ERR_UNSUPPORTED, "rx_mbar_create: out of device memory for u_kn and its reduction buffers");
    }
    if (e != cudaSuccess) MBAR_CREATE_FAIL(RX_ERR_CUDA, std::string("rx_mbar_create: ") + cudaGetErrorString(e));
    h->logN.resize(K);
    h->Nk.resize(K);
    for (int k = 0; k < K; ++k) {
        h->Nk[k] = (double)N_k[k];
        h->logN[k] = N_k[k] > 0 ? log((double)N_k[k]) : -INFINITY;
    }
    h->h_rows.resize(2 * (K + 1));
    h->log_wsum.assign(K, NAN);
    h->h_gram.resize((size_t)h->n_pairs * GT * GT);
    out = std::move(h);
    return RX_OK;
}

// u_kn -= m_n on the handle's stream (k_mbar_shift); d_c holds log N_k until the first run
static cudaError_t mbar_shift(rx_mbar *h) {
    cudaError_t c = cudaMemcpyAsync(h->d_c, h->logN.data(), h->K * sizeof(double), cudaMemcpyHostToDevice, h->stream);
    if (c != cudaSuccess) return c;
    const long long b = std::min(((long long)h->N + 255) / 256, (long long)h->n_sm * 16);
    k_mbar_shift<<<(int)b, 256, 0, h->stream>>>(h->d_u, h->N, h->K, h->d_c, h->d_shift);
    c = cudaGetLastError();
    return c == cudaSuccess ? cudaStreamSynchronize(h->stream) : c;
}

extern "C" int rx_mbar_create_from_history(rx_engine *e, int32_t K, int64_t n_sel, const int64_t *iterations,
                                           const int32_t *columns, const int64_t *N_k, rx_mbar **out) {
    if (!out) MBAR_CREATE_FAIL(RX_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (!e || K < 1 || n_sel < 1 || !iterations || !columns || !N_k)
        MBAR_CREATE_FAIL(RX_ERR_INVALID, "rx_mbar_create_from_history: need an engine, K >= 1, n_sel >= 1, iterations, "
                                         "columns and N_k");
    const int R = e->cfg.n_replicas, W = e->cfg.n_states + e->hist_u;
    for (int64_t j = 0; j < n_sel; ++j)
        if (iterations[j] < 0 || iterations[j] >= e->hist_len)
            MBAR_CREATE_FAIL(RX_ERR_INVALID, "rx_mbar_create_from_history: iteration " + std::to_string(iterations[j]) +
                                                 " is not in the history of " + std::to_string(e->hist_len));
    for (int i = 0; i < K; ++i)
        if (columns[i] < 0 || columns[i] >= W)
            MBAR_CREATE_FAIL(RX_ERR_INVALID, "rx_mbar_create_from_history: column " + std::to_string(columns[i]) +
                                                 " is not in a history row of " + std::to_string(W));
    const int64_t N = (int64_t)R * n_sel;
    const int j_tiles = (int)((n_sel + TT - 1) / TT);
    if ((long long)R * j_tiles > INT32_MAX || (K + TT - 1) / TT > 65535)
        MBAR_CREATE_FAIL(RX_ERR_UNSUPPORTED, "rx_mbar_create_from_history: too many samples or states for one gather");
    if (cudaSetDevice(e->cfg.device) != cudaSuccess) MBAR_CREATE_FAIL(RX_ERR_CUDA, "rx_mbar_create_from_history: cudaSetDevice failed");
    std::unique_ptr<rx_mbar> h;
    int rc = mbar_alloc(K, N, N_k, n_sel * sizeof(long long) + K * sizeof(int) + sizeof(int), h);
    if (rc) return rc;
    DevBuf<long long> d_iter;
    DevBuf<int> d_cols, d_bad;
    cudaError_t c = d_iter.alloc(n_sel);
    if (c == cudaSuccess) c = d_cols.alloc(K);
    if (c == cudaSuccess) c = d_bad.alloc(1);
    // the engine's appends are queued on its stream
    if (c == cudaSuccess) c = cudaStreamSynchronize(e->stream);
    if (c == cudaSuccess) c = cudaMemcpyAsync(d_iter, iterations, n_sel * sizeof(long long), cudaMemcpyHostToDevice, h->stream);
    if (c == cudaSuccess) c = cudaMemcpyAsync(d_cols, columns, K * sizeof(int), cudaMemcpyHostToDevice, h->stream);
    if (c == cudaSuccess) c = cudaMemsetAsync(d_bad, 0, sizeof(int), h->stream);
    if (c == cudaSuccess) {
        k_mbar_gather<<<dim3(R * j_tiles, (K + TT - 1) / TT), dim3(TT, TROWS), 0, h->stream>>>(
            e->d_hist, R, W, d_iter, (int)n_sel, j_tiles, d_cols, K, h->d_u, d_bad);
        c = cudaGetLastError();
    }
    if (c == cudaSuccess) c = mbar_shift(h.get());
    int bad = 0;
    if (c == cudaSuccess) c = cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, h->stream);
    if (c == cudaSuccess) c = cudaStreamSynchronize(h->stream);
    if (c != cudaSuccess) MBAR_CREATE_FAIL(RX_ERR_CUDA, std::string("rx_mbar_create_from_history: ") + cudaGetErrorString(c));
    if (bad) MBAR_CREATE_FAIL(RX_ERR_INVALID, "rx_mbar_create_from_history: u_kn must be finite");
    *out = h.release();
    return RX_OK;
}

extern "C" int rx_mbar_create(int32_t K, int64_t N, const double *u_kn, const int64_t *N_k, rx_mbar **out) {
    if (!out) MBAR_CREATE_FAIL(RX_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (K < 1 || N < 1 || !u_kn || !N_k) MBAR_CREATE_FAIL(RX_ERR_INVALID, "rx_mbar_create: need K >= 1, N >= 1, u_kn and N_k");
    std::unique_ptr<rx_mbar> h;
    int rc = mbar_alloc(K, N, N_k, 0, h);
    if (rc) return rc;
    if (cudaMemcpy(h->d_u, u_kn, (size_t)K * N * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess)
        MBAR_CREATE_FAIL(RX_ERR_CUDA, "rx_mbar_create: upload of u_kn failed");
    if (mbar_shift(h.get()) != cudaSuccess) MBAR_CREATE_FAIL(RX_ERR_CUDA, "rx_mbar_create: shift of u_kn failed");
    *out = h.release();
    return RX_OK;
}
#undef MBAR_CREATE_FAIL

extern "C" void rx_mbar_destroy(rx_mbar *h) { delete h; }

extern "C" int rx_mbar_set_max_blocks(rx_mbar *h, int32_t max_blocks) {
    if (!h || max_blocks < 0) return RX_ERR_INVALID;
    h->max_blocks = max_blocks;
    return RX_OK;
}

extern "C" int rx_mbar_evaluate(rx_mbar *h, const double *f_k, double *logden_sum, double *grad, double *hess) {
    if (!h) return RX_ERR_INVALID;
    if (!f_k) RX_FAIL(h, RX_ERR_INVALID, "f_k is NULL");
    const int rc = run(h, f_k, hess != nullptr);
    if (rc) return rc;
    const int K = h->K;
    const std::vector<double> &Nk = h->Nk, &lw = h->log_wsum;
    if (logden_sum) *logden_sum = h->h_rows[2 * K];
    // N_i - N_i sum_n W_in = -N_i expm1(log sum_n W_in): no cancellation when the sum is far from 1.  Rows and columns of
    // states without samples are 0 (their W at f_i = 0 may be inf).
    if (grad)
        for (int i = 0; i < K; ++i) grad[i] = Nk[i] > 0 ? -Nk[i] * expm1(lw[i]) : 0.0;
    if (hess) {
        unpack_gram(h, hess);
        for (int i = 0; i < K; ++i) {
            for (int j = 0; j < K; ++j)
                hess[(size_t)i * K + j] = Nk[i] > 0 && Nk[j] > 0 ? hess[(size_t)i * K + j] * Nk[i] * Nk[j] : 0.0;
            if (Nk[i] > 0) hess[(size_t)i * K + i] -= Nk[i] * exp(lw[i]);
        }
    }
    return RX_OK;
}

extern "C" int rx_mbar_gram(rx_mbar *h, const double *f_k, double *G, double *wsum) {
    if (!h) return RX_ERR_INVALID;
    if (!f_k || !G) RX_FAIL(h, RX_ERR_INVALID, "f_k and G must not be NULL");
    const int rc = run(h, f_k, true);
    if (rc) return rc;
    unpack_gram(h, G);
    if (wsum)
        for (int i = 0; i < h->K; ++i) wsum[i] = exp(h->log_wsum[i]);
    return RX_OK;
}

extern "C" int rx_mbar_get_log_wsum(rx_mbar *h, double *log_wsum) {
    if (!h) return RX_ERR_INVALID;
    if (!log_wsum) RX_FAIL(h, RX_ERR_INVALID, "log_wsum is NULL");
    memcpy(log_wsum, h->log_wsum.data(), h->K * sizeof(double));
    return RX_OK;
}

extern "C" int rx_mbar_get_logden(rx_mbar *h, double *logD) {
    if (!h) return RX_ERR_INVALID;
    if (!logD) RX_FAIL(h, RX_ERR_INVALID, "logD is NULL");
    RX_CHECK_CUDA(h, cudaSetDevice(h->device));
    // the device holds log D_n of the shifted u_kn, log D_n + m_n
    std::vector<double> m(h->N);
    RX_CHECK_CUDA(h, cudaMemcpy(logD, h->d_logD, h->N * sizeof(double), cudaMemcpyDeviceToHost));
    RX_CHECK_CUDA(h, cudaMemcpy(m.data(), h->d_shift, h->N * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t n = 0; n < h->N; ++n) logD[n] -= m[n];
    return RX_OK;
}
