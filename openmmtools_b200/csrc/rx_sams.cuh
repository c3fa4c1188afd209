// rx_sams.cuh -- SAMSSampler's state jump and online log-weight update on the device (included at the end of rx_mix.cu).
//
// What it replaces (/root/reference/openmmtools/multistate/sams.py):
//   _global_jump            :477-501   log P_k = -u_k + log w_k - logsumexp(.), new state ~ P (numpy RandomState.choice: one
//                                      random_sample() = two MT19937 words, cdf = cumsum(p) / cdf[-1], searchsorted(side='right'))
//   _update_stage           :564-604   two-stage schedule: flatness criteria on the state histogram / logZ
//   _update_logZ_estimates  :606-681   gamma(t); optimal or Rao-Blackwellized increment per replica, in replica order;
//                                      logZ -= logZ[0] in the second stage
//   _update_log_weights     :683-691   log w = log pi - logZ
// One block; the K x M reduced potentials are already on the device (d_u, all-gathered on every rank, so every rank takes the
// same decision -- replicated like the mixing), the uniforms come from the engine's numpy-RandomState MT19937 stream (the stream
// swap-neighbors uses), and logZ / log w / histogram / stage / t0 stay resident between iterations, so a SAMS iteration needs
// no host arithmetic and no host round trip (rx_sams_run_iterations).
//
// Parity.  The arithmetic is f64 in the reference's order where an order is defined (sequential cumsum by one thread, logZ
// increments in replica order), but exp / log / pow are CUDA's, not numpy's, and the logsumexp sum is a fixed tree, not numpy's
// pairwise sum: logZ agrees with the host restatement (multistate/sams.py, itself pinned bit for bit to the reference) to
// ~1e-13 relative, and the jump index is the same unless the uniform falls within ~1e-15 of a cdf boundary.
#pragma once

struct SamsCfg {
    double gamma0, flatness_threshold, beta_factor;
    int method;      // 0 optimal, 1 rao-blackwellized
    int two_stage;   // update_stages == 'two-stage'
    int criteria;    // 0 minimum-visits, 1 histogram-flatness, 2 logZ-flatness
    int pad;
};

struct SamsCtl {      // device-resident scalars
    long long t0;
    long long head;   // words consumed by the last launch
    double gamma;     // gamma of the last update (NaN before the first)
    int stage;
    int pad;
};

struct SamsState {
    SamsCfg cfg;
    int M = 0;
    DevBuf<double> d_logZ, d_log_pi, d_log_w;
    DevBuf<long long> d_hist;
    DevBuf<int> d_prev;   // [K] states before the last jump
    DevBuf<SamsCtl> d_ctl;
};
void RecordDelete::operator()(SamsState *s) const { delete s; }

#define SAMS_THREADS 256

__device__ __forceinline__ double sams_block_reduce(double v, bool is_max, double *scratch) {   // fixed tree; result to all threads
    for (int o = 16; o > 0; o >>= 1) {
        const double w = __shfl_xor_sync(0xffffffffu, v, o);
        v = is_max ? fmax(v, w) : v + w;
    }
    __syncthreads();   // (scratch may still be read from a previous call)
    if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = scratch[0];
    for (int q = 1; q < SAMS_THREADS / 32; q++) r = is_max ? fmax(r, scratch[q]) : r + scratch[q];
    return r;
}

__global__ void __launch_bounds__(SAMS_THREADS) k_sams_step(const uint32_t *__restrict__ words, const double *__restrict__ u, int K,
                                                            int M, int *__restrict__ perm, SamsCfg cfg, double *__restrict__ logZ,
                                                            const double *__restrict__ log_pi, double *__restrict__ log_w,
                                                            long long *__restrict__ hist, SamsCtl *__restrict__ ctl,
                                                            int *__restrict__ prev, long long iteration, int update) {
    extern __shared__ double sams_sh[];
    double *lp = sams_sh, *cdf = sams_sh + M;
    __shared__ double scratch[SAMS_THREADS / 32];
    __shared__ int s_new;
    const int tid = threadIdx.x;
    int stage = ctl->stage;
    long long t0 = ctl->t0;
    double gamma = 0.0;
    if (update) {
        // ---- _update_stage (sams.py:564-604)
        if (cfg.two_stage && stage == 0) {
            double nsum = 0.0, bad = 0.0;     // bad: states that fail the criterion
            for (int l = tid; l < M; l += SAMS_THREADS) nsum += (double)hist[l];
            nsum = sams_block_reduce(nsum, false, scratch);
            if (nsum > 0.0) {
                for (int l = tid; l < M; l += SAMS_THREADS) {
                    bool ok;
                    if (cfg.criteria == 0) ok = hist[l] >= 1;
                    else if (cfg.criteria == 1) { const double pi = exp(log_pi[l]); ok = fabs(pi - (double)hist[l] / nsum) / pi < cfg.flatness_threshold; }
                    else ok = fabs(logZ[l] / cfg.gamma0) > cfg.flatness_threshold;
                    if (!ok) bad += 1.0;
                }
                bad = sams_block_reduce(bad, false, scratch);
                if (bad == 0.0 || (t0 > 0 && iteration > t0)) { stage = 1; t0 = iteration - 1; }
            }
        }
        // ---- gamma (sams.py:627-636)
        double pmin = 1e300;
        for (int l = tid; l < M; l += SAMS_THREADS) pmin = fmin(pmin, exp(log_pi[l]));
        const double pi_star = -sams_block_reduce(-pmin, true, scratch);
        const double t = (double)iteration;
        gamma = stage == 0 ? cfg.gamma0 * fmin(pi_star, pow(t, -cfg.beta_factor))
                           : cfg.gamma0 * fmin(pi_star, 1.0 / (t - (double)t0 + pow((double)t0, cfg.beta_factor)));
    }
    long long p = 0;
    for (int r = 0; r < K; r++) {
        // ---- _global_jump of replica r (sams.py:477-501; the neighbourhood of a global jump is every state)
        const int cur = perm[r];
        double amax = -1e300;
        for (int l = tid; l < M; l += SAMS_THREADS) { const double v = -u[(size_t)r * M + l] + log_w[l]; lp[l] = v; amax = fmax(amax, v); }
        amax = sams_block_reduce(amax, true, scratch);
        double s = 0.0;
        for (int l = tid; l < M; l += SAMS_THREADS) s += exp(lp[l] - amax);
        s = sams_block_reduce(s, false, scratch);
        const double lse = log(s) + amax;
        for (int l = tid; l < M; l += SAMS_THREADS) { const double v = lp[l] - lse; lp[l] = v; cdf[l] = exp(v); }
        __syncthreads();
        if (tid == 0) {
            double c = 0.0;
            for (int l = 0; l < M; l++) { c += cdf[l]; cdf[l] = c; }     // np.cumsum: sequential
            const double U = mt_double(words[p], words[p + 1]);
            int lo = 0, hi = M;                                         // searchsorted(cdf / cdf[-1], U, side='right')
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (cdf[mid] / c <= U) lo = mid + 1; else hi = mid; }
            s_new = lo < M ? lo : M - 1;
            prev[r] = cur;
            perm[r] = s_new;
        }
        p += 2;
        __syncthreads();
        const int nw = s_new;
        // ---- this replica's logZ increment (sams.py:638-676), with the state it has jumped to
        if (update) {
            if (cfg.method == 0) { if (tid == 0) logZ[nw] += gamma * exp(-log_pi[nw]); }
            else for (int l = tid; l < M; l += SAMS_THREADS) logZ[l] += gamma * exp(lp[l] - log_pi[l]);
        }
        __syncthreads();
    }
    if (update) {
        const double z0 = logZ[0];
        __syncthreads();
        for (int l = tid; l < M; l += SAMS_THREADS) {
            const double z = stage == 1 ? logZ[l] - z0 : logZ[l];       // sams.py:678-679
            logZ[l] = z;
            log_w[l] = log_pi[l] - z;                                   // sams.py:683-691
        }
    }
    // the histogram the next _update_stage sees (sams.py:385-393 accumulates it when the iteration is reported)
    if (tid == 0) {
        for (int r = 0; r < K; r++) hist[perm[r]] += 1;
        ctl->stage = stage; ctl->t0 = t0; ctl->head = p;
        if (update) ctl->gamma = gamma;
    }
}

int rxi_sams_set(rx_engine *h, const rx_sams_config *c, const double *log_target, const double *logZ, const int64_t *histogram) {
    const int M = h->cfg.n_states, K = h->cfg.n_replicas;
    if (M > 4096) RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_sams_set: more than 4096 states");
    if (c->weight_update_method < 0 || c->weight_update_method > 1 || c->flatness_criteria < 0 || c->flatness_criteria > 2 ||
        c->stage < 0 || c->stage > 1 || !(c->gamma0 > 0))
        RX_FAIL(h, RX_ERR_INVALID, "rx_sams_set: bad configuration");
    if (!h->sams) {   // taken by the engine once all its buffers exist
        RecordPtr<SamsState> fresh(new SamsState());
        fresh->M = M;
        RX_CHECK_CUDA(h, fresh->d_logZ.alloc(M));
        RX_CHECK_CUDA(h, fresh->d_log_pi.alloc(M));
        RX_CHECK_CUDA(h, fresh->d_log_w.alloc(M));
        RX_CHECK_CUDA(h, fresh->d_hist.alloc(M));
        RX_CHECK_CUDA(h, fresh->d_prev.alloc(K));
        RX_CHECK_CUDA(h, fresh->d_ctl.alloc(1));
        h->sams = std::move(fresh);
    }
    SamsState *s = h->sams.get();
    s->cfg = SamsCfg{c->gamma0, c->flatness_threshold, 0.8, c->weight_update_method, c->two_stage ? 1 : 0, c->flatness_criteria, 0};
    std::vector<double> lw(M);
    std::vector<long long> hh(M, 0);
    for (int l = 0; l < M; l++) { lw[l] = log_target[l] - logZ[l]; if (histogram) hh[l] = histogram[l]; }
    SamsCtl ctl = {c->t0, 0, nan(""), c->stage, 0};
    RX_CHECK_CUDA(h, cudaMemcpyAsync(s->d_logZ, logZ, sizeof(double) * M, cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(s->d_log_pi, log_target, sizeof(double) * M, cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(s->d_log_w, lw.data(), sizeof(double) * M, cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(s->d_hist, hh.data(), sizeof(long long) * M, cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(s->d_ctl, &ctl, sizeof(ctl), cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaMemsetAsync(s->d_prev, 0, sizeof(int) * K, h->stream));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return RX_OK;
}

int rxi_sams_set_histogram(rx_engine *h, const int64_t *histogram) {
    const SamsState *s = h->sams.get();
    if (!s) RX_FAIL(h, RX_ERR_INVALID, "rx_sams_step: rx_sams_set must be called first");
    RX_CHECK_CUDA(h, cudaMemcpyAsync(s->d_hist, histogram, sizeof(long long) * s->M, cudaMemcpyHostToDevice, h->stream));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));   // (the caller's buffer may be pageable and short-lived)
    return RX_OK;
}

// one jump (+ update) on the engine's stream; no host synchronisation
int rxi_sams_step(rx_engine *h, long long iteration, int update, int *launches) {
    const SamsState *s = h->sams.get();
    if (!s) RX_FAIL(h, RX_ERR_INVALID, "rx_sams_step: rx_sams_set must be called first");
    MTStream &S = h->streams[RX_STREAM_NUMPY];
    if (!S.seeded) RX_FAIL(h, RX_ERR_INVALID, "rx_sams_step: the numpy MT19937 stream has not been seeded (rx_mix_seed)");
    const int K = h->cfg.n_replicas, M = h->cfg.n_states;
    int rc = stream_fill(h, S, (size_t)2 * K + 64, launches, h->stream);
    if (rc) return rc;
    const size_t smem = 2 * (size_t)M * sizeof(double);
    if (smem > 48 * 1024) RX_CHECK_CUDA(h, cudaFuncSetAttribute(k_sams_step, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_sams_step<<<1, SAMS_THREADS, smem, h->stream>>>(S.d_words, h->d_u, K, M, h->d_perm, s->cfg, s->d_logZ, s->d_log_pi, s->d_log_w,
                                                      s->d_hist, s->d_ctl, s->d_prev, iteration, update);
    RX_CHECK_CUDA(h, cudaGetLastError());
    (*launches)++;
    return stream_consume(h, S, (size_t)2 * K, launches);   // (one uniform per replica: known without reading the device)
}

int rxi_sams_get(rx_engine *h, double *logZ, double *log_weights, int64_t *histogram, int32_t *stage, int64_t *t0, double *gamma,
                 int64_t *states, int64_t *previous_states) {
    const SamsState *s = h->sams.get();
    if (!s) RX_FAIL(h, RX_ERR_INVALID, "rx_sams_get: rx_sams_set must be called first");
    const int M = s->M, K = h->cfg.n_replicas;
    SamsCtl ctl;
    std::vector<int> a(K), b(K);
    if (logZ) RX_CHECK_CUDA(h, cudaMemcpyAsync(logZ, s->d_logZ, sizeof(double) * M, cudaMemcpyDeviceToHost, h->stream));
    if (log_weights) RX_CHECK_CUDA(h, cudaMemcpyAsync(log_weights, s->d_log_w, sizeof(double) * M, cudaMemcpyDeviceToHost, h->stream));
    if (histogram) RX_CHECK_CUDA(h, cudaMemcpyAsync(histogram, s->d_hist, sizeof(long long) * M, cudaMemcpyDeviceToHost, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(&ctl, s->d_ctl, sizeof(ctl), cudaMemcpyDeviceToHost, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(a.data(), h->d_perm, sizeof(int) * K, cudaMemcpyDeviceToHost, h->stream));
    RX_CHECK_CUDA(h, cudaMemcpyAsync(b.data(), s->d_prev, sizeof(int) * K, cudaMemcpyDeviceToHost, h->stream));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (stage) *stage = ctl.stage;
    if (t0) *t0 = ctl.t0;
    if (gamma) *gamma = ctl.gamma;
    for (int k = 0; k < K; k++) { if (states) states[k] = a[k]; if (previous_states) previous_states[k] = b[k]; }
    return RX_OK;
}
