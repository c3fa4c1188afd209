// rx_api.cu -- the C ABI of librx_b200.so (include/rx_b200.h): lifecycle, tables, replica I/O, phase calls,
// the fused iteration loop, NCCL (dlopen) energy-row all-gather.
#include "rx_internal.cuh"
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <algorithm>

thread_local std::string g_rx_create_error;

extern "C" int rx_abi_version(void) { return RX_ABI_VERSION; }

extern "C" const char *rx_last_error(const rx_engine *h) { return h ? h->err.c_str() : g_rx_create_error.c_str(); }

#define CREATE_FAIL(code, msg)       \
    do {                             \
        g_rx_create_error = (msg);   \
        if (h) rx_destroy(h);        \
        return (code);               \
    } while (0)
#define CREATE_CUDA(call)                                                                 \
    do {                                                                                  \
        cudaError_t _e = (call);                                                          \
        if (_e != cudaSuccess) CREATE_FAIL(RX_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
    } while (0)

extern "C" int rx_create(const rx_config *cfg, rx_engine **out) {
    rx_engine *h = nullptr;
    if (!cfg || !out) CREATE_FAIL(RX_ERR_INVALID, "rx_create: null argument");
    if (cfg->abi_version != RX_ABI_VERSION) CREATE_FAIL(RX_ERR_INVALID, "rx_create: ABI version mismatch");
    if (cfg->n_replicas < 1 || cfg->n_states < 1) CREATE_FAIL(RX_ERR_INVALID, "rx_create: n_replicas and n_states must be >= 1");
    if (cfg->system_kind < RX_SYSTEM_NONE || cfg->system_kind > RX_SYSTEM_MOLECULE) CREATE_FAIL(RX_ERR_INVALID, "rx_create: unknown system_kind");
    if (cfg->system_kind != RX_SYSTEM_NONE && cfg->n_atoms < 1) CREATE_FAIL(RX_ERR_INVALID, "rx_create: n_atoms must be >= 1");
    if (cfg->system_kind == RX_SYSTEM_MOLECULE && cfg->n_atoms > 32) CREATE_FAIL(RX_ERR_UNSUPPORTED, "rx_create: a molecule has at most 32 atoms");
    if (cfg->world_size < 1 || cfg->rank < 0 || cfg->rank >= cfg->world_size) CREATE_FAIL(RX_ERR_INVALID, "rx_create: bad rank/world_size");
    if (cfg->system_kind == RX_SYSTEM_LJ_ALCH) {
        for (int d = 0; d < 3; d++)
            if (!(cfg->box[d] > 0) || cfg->r_cutoff > 0.5 * cfg->box[d])
                CREATE_FAIL(RX_ERR_INVALID, "rx_create: cutoff must not exceed half the box edge (minimum image)");
        if (!(cfg->r_cutoff > 0)) CREATE_FAIL(RX_ERR_INVALID, "rx_create: r_cutoff must be > 0");
        if (cfg->use_switch && !(cfg->r_switch >= 0 && cfg->r_switch < cfg->r_cutoff))
            CREATE_FAIL(RX_ERR_INVALID, "rx_create: need 0 <= r_switch < r_cutoff");
        if (!(cfg->softcore_c > 0)) CREATE_FAIL(RX_ERR_INVALID, "rx_create: softcore_c must be > 0");
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) CREATE_FAIL(RX_ERR_CUDA, std::string("rx_create: no CUDA device available (") + cudaGetErrorString(e) + "); this engine has no CPU fallback");
    if (cfg->device < 0 || cfg->device >= ndev) CREATE_FAIL(RX_ERR_INVALID, "rx_create: device ordinal out of range");
    CREATE_CUDA(cudaSetDevice(cfg->device));
    h = new rx_engine();
    h->cfg = *cfg;
    CREATE_CUDA(cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, cfg->device));
    CREATE_CUDA(cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, cfg->device));
    const int K = cfg->n_replicas, M = cfg->n_states, N = cfg->n_atoms, W = cfg->world_size, R = cfg->rank;
    h->k0 = (int)(((long long)R * K) / W);
    h->kloc = (int)(((long long)(R + 1) * K) / W) - h->k0;
    {
        // The side stream prepares the NEXT mixing call (random words, slot records) while the replicas propagate on the main
        // stream: it gets the lowest priority, so that its thread blocks only fill what k_propagate leaves free.
        int prio_lo = 0, prio_hi = 0;
        CREATE_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
        CREATE_CUDA(cudaStreamCreateWithPriority(&h->stream, cudaStreamNonBlocking, prio_hi));
        CREATE_CUDA(cudaStreamCreateWithPriority(&h->stream_rng, cudaStreamNonBlocking, prio_lo));
    }
    for (int i = 0; i < 8; i++) CREATE_CUDA(cudaEventCreate(&h->ev[i]));
    for (int i = 0; i < 2; i++) CREATE_CUDA(cudaEventCreate(&h->ev_user[i]));
    for (int i = 0; i < 2; i++) CREATE_CUDA(cudaEventCreate(&h->ev_walk[i]));
    CREATE_CUDA(cudaEventCreateWithFlags(&h->ev_prepared, cudaEventDisableTiming));
    CREATE_CUDA(cudaEventCreateWithFlags(&h->ev_consumed, cudaEventDisableTiming));
    CREATE_CUDA(h->d_perm.alloc(K));
    CREATE_CUDA(h->d_u.alloc((size_t)K * M));
    CREATE_CUDA(cudaMemset(h->d_u, 0, sizeof(double) * (size_t)K * M));
    CREATE_CUDA(h->d_nacc.alloc((size_t)M * M));
    CREATE_CUDA(h->d_nprop.alloc((size_t)M * M));
    CREATE_CUDA(cudaMemset(h->d_nacc, 0, sizeof(unsigned long long) * (size_t)M * M));
    CREATE_CUDA(cudaMemset(h->d_nprop, 0, sizeof(unsigned long long) * (size_t)M * M));
    CREATE_CUDA(h->d_pot.alloc(K));
    CREATE_CUDA(h->d_kin.alloc(K));
    CREATE_CUDA(cudaMemset(h->d_pot, 0, sizeof(double) * K));
    CREATE_CUDA(cudaMemset(h->d_kin, 0, sizeof(double) * K));
    CREATE_CUDA(h->d_nan.alloc(K));
    CREATE_CUDA(cudaMemset(h->d_nan, 0, sizeof(int) * K));
    CREATE_CUDA(h->d_err.alloc(1));
    CREATE_CUDA(cudaMemset(h->d_err, 0, sizeof(int)));
    CREATE_CUDA(h->d_ctl.alloc(1));
    CREATE_CUDA(h->d_states.alloc(M));
    {
        std::vector<int> perm(K);
        for (int k = 0; k < K; k++) perm[k] = k % M;
        CREATE_CUDA(cudaMemcpy(h->d_perm, perm.data(), sizeof(int) * K, cudaMemcpyHostToDevice));
    }
    if (cfg->system_kind != RX_SYSTEM_NONE) {
        const size_t n = (size_t)(h->kloc > 0 ? h->kloc : 1) * N;
        // (a molecule keeps its state as double[3] per atom, the other systems as float4)
        const size_t per_atom = cfg->system_kind == RX_SYSTEM_MOLECULE ? 3 * sizeof(double) : sizeof(float4);
        CREATE_CUDA(h->d_pos.alloc(n, per_atom));
        CREATE_CUDA(h->d_vel.alloc(n, per_atom));
        CREATE_CUDA(cudaMemset(h->d_pos, 0, per_atom * n));
        CREATE_CUDA(cudaMemset(h->d_vel, 0, per_atom * n));
        CREATE_CUDA(h->d_io.alloc(3 * n));
        CREATE_CUDA(h->h_io.alloc(3 * n));
        CREATE_CUDA(h->d_atom.alloc(N));
        CREATE_CUDA(h->d_atom_d.alloc(N));
        CREATE_CUDA(h->d_alch_list.alloc(N));
    }
    *out = h;
    return RX_OK;
}

// The engine's device and pinned memory is freed with it (CudaBuf, RecordPtr); streams, events, NCCL and the caller's pinned
// buffers are released here.
extern "C" void rx_destroy(rx_engine *h) {
    if (!h) return;
    cudaSetDevice(h->cfg.device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->stream_rng) cudaStreamSynchronize(h->stream_rng);
    if (h->ev_prepared) cudaEventDestroy(h->ev_prepared);
    if (h->ev_consumed) cudaEventDestroy(h->ev_consumed);
    if (h->nccl_comm && h->nccl_lib) {
        typedef int (*destroy_t)(void *);
        destroy_t f = (destroy_t)dlsym(h->nccl_lib, "ncclCommDestroy");
        if (f) f(h->nccl_comm);
    }
    for (int i = 0; i < 8; i++) if (h->ev[i]) cudaEventDestroy(h->ev[i]);
    for (int i = 0; i < 2; i++) if (h->ev_user[i]) cudaEventDestroy(h->ev_user[i]);
    for (int i = 0; i < 2; i++) if (h->ev_walk[i]) cudaEventDestroy(h->ev_walk[i]);
    for (const auto &r : h->pinned) cudaHostUnregister((void *)r.first);
    if (h->stream) cudaStreamDestroy(h->stream);
    if (h->stream_rng) cudaStreamDestroy(h->stream_rng);
    delete h;
}

#define ENTER(h)                                  \
    if (!(h)) return RX_ERR_INVALID;              \
    (h)->err.clear();                             \
    RX_CHECK_CUDA(h, cudaSetDevice((h)->cfg.device))

static int upload_atoms(rx_engine *h, const std::vector<int> &al);

extern "C" int rx_set_particles(rx_engine *h, const double *sigma, const double *epsilon, const double *mass,
                                const uint8_t *alch) {
    ENTER(h);
    if (h->cfg.system_kind == RX_SYSTEM_NONE) RX_FAIL(h, RX_ERR_INVALID, "rx_set_particles: engine has no particle system");
    if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) RX_FAIL(h, RX_ERR_INVALID, "rx_set_particles: use rx_set_molecule for RX_SYSTEM_MOLECULE");
    if (!mass) RX_FAIL(h, RX_ERR_INVALID, "rx_set_particles: mass is required");
    const int N = h->cfg.n_atoms;
    const bool lj = h->cfg.system_kind == RX_SYSTEM_LJ_ALCH;
    if (lj && (!sigma || !epsilon)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_particles: sigma and epsilon are required");
    std::vector<float4> a(N);
    std::vector<double4> ad(N);
    std::vector<int> al;
    for (int i = 0; i < N; i++) {
        const double s = lj ? sigma[i] : 1.0, e = lj ? epsilon[i] : 0.0, m = mass[i];
        const bool isal = lj && alch && alch[i];
        if (!(m > 0)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_particles: masses must be > 0");
        if (lj && (!(s > 0) || e < 0)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_particles: need sigma > 0 and epsilon >= 0");
        a[i] = make_float4((float)s, (float)sqrt(e), (float)(1.0 / m), isal ? 1.f : 0.f);
        ad[i] = make_double4(s, e, m, isal ? 1.0 : 0.0);
        if (isal) al.push_back(i);
    }
    h->have_particles = false;
    h->two_regions = false;
    h->annihilate_mask = 0;
    h->h_atom = a;
    h->h_atom_d = ad;
    return upload_atoms(h, al);
}

// The atom tables of h_atom / h_atom_d, the list `al` of alchemical atoms and the pair scratch sized for it.
static int upload_atoms(rx_engine *h, const std::vector<int> &al) {
    const int N = h->cfg.n_atoms;
    h->n_alch = (int)al.size();
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_atom, h->h_atom.data(), sizeof(float4) * N, cudaMemcpyHostToDevice));
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_atom_d, h->h_atom_d.data(), sizeof(double4) * N, cudaMemcpyHostToDevice));
    if (h->n_alch) RX_CHECK_CUDA(h, cudaMemcpy(h->d_alch_list, al.data(), sizeof(int) * h->n_alch, cudaMemcpyHostToDevice));
    // scratch for the lambda-controlled pair list of each owned replica
    long long cap = (long long)h->n_alch * (N - 1);
    if (cap > (1 << 18)) cap = 1 << 18;
    if (cap < 1) cap = 1;
    RX_CHECK_CUDA(h, h->d_pairs.alloc((size_t)cap * (h->kloc > 0 ? h->kloc : 1)));
    h->pair_cap = (int)cap;
    h->have_particles = true;
    return RX_OK;
}

extern "C" int rx_set_alchemical_regions(rx_engine *h, const uint8_t *region, int32_t annihilate_1, int32_t annihilate_2) {
    ENTER(h);
    if (h->cfg.system_kind != RX_SYSTEM_LJ_ALCH) RX_FAIL(h, RX_ERR_INVALID, "rx_set_alchemical_regions: RX_SYSTEM_LJ_ALCH engines only");
    if (!region) RX_FAIL(h, RX_ERR_INVALID, "rx_set_alchemical_regions: null");
    if (h->h_atom.empty()) RX_FAIL(h, RX_ERR_INVALID, "rx_set_alchemical_regions: call rx_set_particles first");
    const int N = h->cfg.n_atoms;
    for (int i = 0; i < N; i++)
        if (region[i] > 2) RX_FAIL(h, RX_ERR_INVALID, "rx_set_alchemical_regions: region ids are 0 (environment), 1 or 2");
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    std::vector<int> al;
    for (int i = 0; i < N; i++) {
        h->h_atom[i].w = (float)region[i];
        h->h_atom_d[i].w = (double)region[i];
        if (region[i]) al.push_back(i);
    }
    h->have_particles = false;
    h->two_regions = true;
    h->annihilate_mask = (annihilate_1 ? 1 : 0) | (annihilate_2 ? 2 : 0);
    return upload_atoms(h, al);
}

extern "C" int rx_set_molecule(rx_engine *h, const rx_molecule *molecule) {
    ENTER(h);
    if (h->cfg.system_kind != RX_SYSTEM_MOLECULE) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: the engine was not created with RX_SYSTEM_MOLECULE");
    if (!molecule) RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: null");
    if (molecule->n_bonds < 0 || molecule->n_angles < 0 || molecule->n_torsions < 0 || molecule->n_exclusions < 0 ||
        molecule->n_exceptions < 0 || molecule->n_constraints < 0)
        RX_FAIL(h, RX_ERR_INVALID, "rx_set_molecule: negative count");
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return rxi_set_molecule(h, molecule);
}

extern "C" int rx_set_implicit_solvent(rx_engine *h, const rx_gbsa *gbsa) {
    ENTER(h);
    if (h->cfg.system_kind != RX_SYSTEM_MOLECULE) RX_FAIL(h, RX_ERR_INVALID, "rx_set_implicit_solvent: the engine was not created with RX_SYSTEM_MOLECULE");
    if (!gbsa) RX_FAIL(h, RX_ERR_INVALID, "rx_set_implicit_solvent: null");
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return rxi_set_implicit_solvent(h, gbsa);
}

static int convert_states(rx_engine *h, const rx_state_params *s, int n, std::vector<StateDev> &out, const char *who) {
    out.resize(n);
    for (int l = 0; l < n; l++) {
        if (!(s[l].temperature > 0)) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": temperature must be > 0");
        if (h->cfg.system_kind == RX_SYSTEM_LJ_ALCH && !(s[l].lambda_sterics >= 0.0 && s[l].lambda_sterics <= 1.0))
            RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": lambda_sterics must be in [0, 1]");
        if (h->cfg.system_kind == RX_SYSTEM_MOLECULE &&
            !(s[l].lambda_sterics >= 0.0 && s[l].lambda_sterics <= 1.0 && s[l].lambda_electrostatics >= 0.0 && s[l].lambda_electrostatics <= 1.0))
            RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": lambda_sterics and lambda_electrostatics must be in [0, 1]");
        StateDev &d = out[l];
        d.kT = RX_KB * s[l].temperature;
        d.beta = 1.0 / d.kT;
        d.lambda = s[l].lambda_sterics;
        d.la = pow(s[l].lambda_sterics, h->cfg.softcore_a);
        d.ob = h->cfg.softcore_alpha * pow(1.0 - s[l].lambda_sterics, h->cfg.softcore_b);
        d.offset = s[l].energy_offset;
        d.ho_K = s[l].ho_K;
        for (int q = 0; q < 3; q++) d.ho_x0[q] = s[l].ho_x0[q];
        d.lambda2 = 1.0; d.la2 = 1.0; d.ob2 = 0.0;
        d.lambda_e = s[l].lambda_electrostatics;
    }
    return RX_OK;
}

// The second region's lambda_sterics of n converted states (`lambda2` may be NULL: 1 everywhere).
static int convert_states_region2(rx_engine *h, const double *lambda2, int n, std::vector<StateDev> &out, const char *who) {
    if (!lambda2) return RX_OK;
    if (h->cfg.system_kind != RX_SYSTEM_LJ_ALCH) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": RX_SYSTEM_LJ_ALCH engines only");
    for (int l = 0; l < n; l++) {
        if (!(lambda2[l] >= 0.0 && lambda2[l] <= 1.0)) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": lambda_sterics must be in [0, 1]");
        StateDev &d = out[l];
        d.lambda2 = lambda2[l];
        d.la2 = pow(lambda2[l], h->cfg.softcore_a);
        d.ob2 = h->cfg.softcore_alpha * pow(1.0 - lambda2[l], h->cfg.softcore_b);
    }
    return RX_OK;
}

extern "C" int rx_set_states_region2(rx_engine *h, const double *lambda2) {
    ENTER(h);
    if (!lambda2) RX_FAIL(h, RX_ERR_INVALID, "rx_set_states_region2: null");
    if (!h->have_states) RX_FAIL(h, RX_ERR_INVALID, "rx_set_states_region2: call rx_set_states first");
    const int M = h->cfg.n_states;
    std::vector<StateDev> tab = h->h_states;
    int rc = convert_states_region2(h, lambda2, M, tab, "rx_set_states_region2");
    if (rc) return rc;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_states, tab.data(), sizeof(StateDev) * M, cudaMemcpyHostToDevice));
    h->h_states = tab;
    return RX_OK;
}

extern "C" int rx_set_states(rx_engine *h, const rx_state_params *s) {
    ENTER(h);
    if (!s) RX_FAIL(h, RX_ERR_INVALID, "rx_set_states: null");
    const int M = h->cfg.n_states;
    int rc = convert_states(h, s, M, h->h_states, "rx_set_states");
    if (rc) return rc;
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_states, h->h_states.data(), sizeof(StateDev) * M, cudaMemcpyHostToDevice));
    h->have_states = true;
    return RX_OK;
}

extern "C" int rx_set_integrator(rx_engine *h, double timestep, double collision_rate, int32_t n_steps,
                                 const char *splitting) {
    ENTER(h);
    if (!(timestep > 0) || collision_rate < 0 || n_steps < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_set_integrator: bad timestep/collision_rate/n_steps");
    if (!splitting) RX_FAIL(h, RX_ERR_INVALID, "rx_set_integrator: null splitting");
    const size_t n = strlen(splitting);
    if (n == 0 || n >= RX_MAX_PROGRAM) RX_FAIL(h, RX_ERR_INVALID, "rx_set_integrator: splitting must have 1..31 substeps");
    bool hasV = false, hasR = false, hasO = false;
    for (size_t i = 0; i < n; i++) {
        const char c = splitting[i];
        if (c == 'V') hasV = true; else if (c == 'R') hasR = true; else if (c == 'O') hasO = true;
        else RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_set_integrator: only R, V and O substeps are supported (no force groups / Metropolization)");
    }
    if (!(hasV && hasR && hasO)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_integrator: splitting must contain R, V and O (integrators.py:1360-1363)");
    h->dt = timestep; h->gamma = collision_rate; h->n_steps = n_steps;
    memset(h->program, 0, sizeof(h->program));
    memcpy(h->program, splitting, n);
    h->have_integrator = true;
    h->hmc = false;
    h->state_moves.clear();   // one move for every state again
    return RX_OK;
}

// The HMC counters and last-trial energies of the owned replicas, allocated (zero) by the first HMC setter.
static int hmc_buffers(rx_engine *h) {
    if (h->d_hmc_stats) return RX_OK;
    const size_t n = (size_t)(h->kloc > 0 ? h->kloc : 1);
    DevBuf<ulonglong2> stats;
    DevBuf<double2> energy;
    RX_CHECK_CUDA(h, stats.alloc(n));
    RX_CHECK_CUDA(h, energy.alloc(n));
    RX_CHECK_CUDA(h, cudaMemset(stats, 0, sizeof(ulonglong2) * n));
    RX_CHECK_CUDA(h, cudaMemset(energy, 0xff, sizeof(double2) * n));   // (NaN: no trial yet)
    h->d_hmc_stats = std::move(stats); h->d_hmc_energy = std::move(energy);
    return RX_OK;
}

static int hmc_check(rx_engine *h, double timestep, int32_t n_steps, const char *who) {
    if (!(timestep > 0) || !isfinite(timestep) || n_steps < 0) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": need timestep > 0 and n_steps >= 0");
    if (h->cfg.system_kind == RX_SYSTEM_NONE) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": engine has no particle system");
    if (h->npt) RX_FAIL(h, RX_ERR_UNSUPPORTED, std::string(who) + ": hybrid Monte Carlo at constant pressure is not provided");
    return hmc_buffers(h);
}

extern "C" int rx_set_hmc_integrator(rx_engine *h, double timestep, int32_t n_steps) {
    ENTER(h);
    int rc = hmc_check(h, timestep, n_steps, "rx_set_hmc_integrator");
    if (rc) return rc;
    h->dt = timestep; h->gamma = 0.0; h->n_steps = n_steps;
    memset(h->program, 0, sizeof(h->program));
    memcpy(h->program, "VRV", 3);
    h->have_integrator = true;
    h->hmc = true;
    h->state_moves.clear();
    return RX_OK;
}

extern "C" int rx_set_state_hmc_integrator(rx_engine *h, int32_t state, double timestep, int32_t n_steps) {
    ENTER(h);
    if (!h->have_integrator || !h->hmc) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_hmc_integrator: rx_set_hmc_integrator must be called first");
    if (state < 0 || state >= h->cfg.n_states) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_hmc_integrator: state out of range");
    int rc = hmc_check(h, timestep, n_steps, "rx_set_state_hmc_integrator");
    if (rc) return rc;
    if (h->state_moves.empty()) {   // start from the common move
        h->state_moves.resize((size_t)h->cfg.n_states);
        for (auto &m : h->state_moves) {
            m.dt = h->dt; m.gamma = 0.0; m.n_steps = h->n_steps; m.reassign = 0; m.hmc = true;
            memcpy(m.program, h->program, sizeof(m.program));
        }
    }
    rx_state_move &m = h->state_moves[(size_t)state];
    m.dt = timestep; m.gamma = 0.0; m.n_steps = n_steps; m.reassign = 0; m.set = true; m.hmc = true;
    memset(m.program, 0, sizeof(m.program));
    memcpy(m.program, "VRV", 3);
    h->state_moves_dirty = true;
    return RX_OK;
}

// Per owned replica: [k0, k0 + kloc) of the [K] arrays; the other entries are left alone.
extern "C" int rx_get_hmc_statistics(rx_engine *h, int64_t *accepted, int64_t *trials) {
    ENTER(h);
    if (!accepted || !trials) RX_FAIL(h, RX_ERR_INVALID, "rx_get_hmc_statistics: null argument");
    const int K = h->cfg.n_replicas;
    for (int k = 0; k < K; k++) if (k < h->k0 || k >= h->k0 + h->kloc) accepted[k] = trials[k] = 0;
    if (!h->d_hmc_stats || h->kloc == 0) {
        for (int k = h->k0; k < h->k0 + h->kloc; k++) accepted[k] = trials[k] = 0;
        return RX_OK;
    }
    std::vector<ulonglong2> c((size_t)h->kloc);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(c.data(), h->d_hmc_stats, sizeof(ulonglong2) * h->kloc, cudaMemcpyDeviceToHost));
    for (int r = 0; r < h->kloc; r++) { accepted[h->k0 + r] = (int64_t)c[r].x; trials[h->k0 + r] = (int64_t)c[r].y; }
    return RX_OK;
}

extern "C" int rx_set_hmc_statistics(rx_engine *h, const int64_t *accepted, const int64_t *trials) {
    ENTER(h);
    if (!accepted || !trials) RX_FAIL(h, RX_ERR_INVALID, "rx_set_hmc_statistics: null argument");
    if (!h->d_hmc_stats) RX_FAIL(h, RX_ERR_INVALID, "rx_set_hmc_statistics: call rx_set_hmc_integrator first");
    std::vector<ulonglong2> c((size_t)h->kloc);
    for (int r = 0; r < h->kloc; r++) {
        const int64_t a = accepted[h->k0 + r], n = trials[h->k0 + r];
        if (a < 0 || n < a) RX_FAIL(h, RX_ERR_INVALID, "rx_set_hmc_statistics: need 0 <= accepted <= trials");
        c[r] = make_ulonglong2((unsigned long long)a, (unsigned long long)n);
    }
    if (h->kloc == 0) return RX_OK;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_hmc_stats, c.data(), sizeof(ulonglong2) * h->kloc, cudaMemcpyHostToDevice));
    return RX_OK;
}

extern "C" int rx_get_hmc_energies(rx_engine *h, double *e_old, double *e_new) {
    ENTER(h);
    if (!e_old || !e_new) RX_FAIL(h, RX_ERR_INVALID, "rx_get_hmc_energies: null argument");
    const int K = h->cfg.n_replicas;
    for (int k = 0; k < K; k++) e_old[k] = e_new[k] = NAN;
    if (!h->d_hmc_energy || h->kloc == 0) return RX_OK;
    std::vector<double2> e((size_t)h->kloc);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(e.data(), h->d_hmc_energy, sizeof(double2) * h->kloc, cudaMemcpyDeviceToHost));
    for (int r = 0; r < h->kloc; r++) { e_old[h->k0 + r] = e[r].x; e_new[h->k0 + r] = e[r].y; }
    return RX_OK;
}

/* One MCMCMove per thermodynamic state (openmmtools/multistate/multistatesampler.py:906-910; a replica is propagated with
 * the move of the state it is in, :1311-1322).  Call after rx_set_integrator (which provides the move of every state not
 * set here) for each state whose move differs; rx_set_integrator again returns to one move for all states. */
extern "C" int rx_set_state_integrator(rx_engine *h, int32_t state, double timestep, double collision_rate, int32_t n_steps,
                                       const char *splitting, int32_t reassign_velocities) {
    ENTER(h);
    if (!h->have_integrator) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_integrator: rx_set_integrator must be called first");
    if (state < 0 || state >= h->cfg.n_states) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_integrator: state out of range");
    if (!(timestep > 0) || collision_rate < 0 || n_steps < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_integrator: bad timestep/collision_rate/n_steps");
    if (!splitting) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_integrator: null splitting");
    const size_t n = strlen(splitting);
    if (n == 0 || n >= RX_MAX_PROGRAM) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_integrator: splitting must have 1..31 substeps");
    bool hasV = false, hasR = false, hasO = false;
    for (size_t i = 0; i < n; i++) {
        const char c = splitting[i];
        if (c == 'V') hasV = true; else if (c == 'R') hasR = true; else if (c == 'O') hasO = true;
        else RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_set_state_integrator: only R, V and O substeps are supported");
    }
    if (!(hasV && hasR && hasO)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_integrator: splitting must contain R, V and O");
    if (h->state_moves.empty()) {   // start from the common move
        h->state_moves.resize((size_t)h->cfg.n_states);
        for (auto &m : h->state_moves) {
            m.dt = h->dt; m.gamma = h->gamma; m.n_steps = h->n_steps; m.reassign = 0; m.hmc = h->hmc;
            memcpy(m.program, h->program, sizeof(m.program));
        }
    }
    rx_state_move &m = h->state_moves[(size_t)state];
    m.dt = timestep; m.gamma = collision_rate; m.n_steps = n_steps; m.reassign = reassign_velocities ? 1 : 0; m.set = true; m.hmc = false;
    memset(m.program, 0, sizeof(m.program));
    memcpy(m.program, splitting, n);
    h->state_moves_dirty = true;
    return RX_OK;
}

// ---- Monte Carlo moves (rx_mc.cuh) ----------------------------------------------------------------------------------------
// Every state's move table on the device, and the number of launches it takes (the most moves any state has).
static int upload_mc_moves(rx_engine *h) {
    const int M = h->cfg.n_states;
    h->mc_slots = 0;
    for (int l = 0; l < M; l++)
        for (int j = 0; j < RX_MAX_MC_MOVES; j++)
            if (h->mc_moves[(size_t)l * RX_MAX_MC_MOVES + j].kind >= 0) h->mc_slots = std::max(h->mc_slots, j + 1);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_mc_moves, h->mc_moves.data(), sizeof(rx_mc_move) * h->mc_moves.size(), cudaMemcpyHostToDevice));
    return RX_OK;
}

extern "C" int rx_set_mc_subsets(rx_engine *h, const int32_t *atoms, int32_t n) {
    ENTER(h);
    if (h->cfg.system_kind == RX_SYSTEM_NONE) RX_FAIL(h, RX_ERR_INVALID, "rx_set_mc_subsets: engine has no particle system");
    if (n < 0 || (n > 0 && !atoms)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_mc_subsets: bad arguments");
    for (int q = 0; q < n; q++)
        if (atoms[q] < 0 || atoms[q] >= h->cfg.n_atoms) RX_FAIL(h, RX_ERR_INVALID, "rx_set_mc_subsets: atom index out of range");
    const size_t mm = (size_t)h->cfg.n_states * RX_MAX_MC_MOVES;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    DevBuf<int32_t> d_atoms;
    RX_CHECK_CUDA(h, d_atoms.alloc(n > 0 ? n : 1));
    if (n > 0) RX_CHECK_CUDA(h, cudaMemcpy(d_atoms, atoms, sizeof(int32_t) * n, cudaMemcpyHostToDevice));
    if (!h->d_mc_moves) {   // the move table and its statistics, taken by the engine once all of them exist
        DevBuf<rx_mc_move> d_moves;
        DevBuf<unsigned long long> d_acc, d_prop;
        DevBuf<double> d_du;
        const size_t nd = (size_t)(h->kloc > 0 ? h->kloc : 1) * RX_MAX_MC_MOVES;
        RX_CHECK_CUDA(h, d_moves.alloc(mm));
        RX_CHECK_CUDA(h, d_acc.alloc(mm));
        RX_CHECK_CUDA(h, d_prop.alloc(mm));
        RX_CHECK_CUDA(h, d_du.alloc(nd));
        RX_CHECK_CUDA(h, cudaMemset(d_acc, 0, sizeof(unsigned long long) * mm));
        RX_CHECK_CUDA(h, cudaMemset(d_prop, 0, sizeof(unsigned long long) * mm));
        RX_CHECK_CUDA(h, cudaMemset(d_du, 0xff, sizeof(double) * nd));   // (NaN: no proposal yet)
        h->d_mc_moves = std::move(d_moves); h->d_mc_du = std::move(d_du);
        h->d_mc_acc = std::move(d_acc); h->d_mc_prop = std::move(d_prop);
    }
    h->d_mc_atoms = std::move(d_atoms);
    h->mc_atoms.assign(atoms, atoms + n);
    rx_mc_move none;
    memset(&none, 0, sizeof(none));
    none.kind = -1;
    h->mc_moves.assign(mm, none);
    return upload_mc_moves(h);
}

extern "C" int rx_set_state_mc_moves(rx_engine *h, int32_t state, int32_t n, const rx_mc_move *moves) {
    ENTER(h);
    const int M = h->cfg.n_states, N = h->cfg.n_atoms;
    if (!h->d_mc_moves) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: call rx_set_mc_subsets first");
    if (state < -1 || state >= M) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: state out of range");
    if (n < 0 || n > RX_MAX_MC_MOVES || (n > 0 && !moves))
        RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: a state has 0 to RX_MAX_MC_MOVES (4) moves");
    if (n > 0 && h->cfg.system_kind == RX_SYSTEM_LJ_ALCH && N > 4096)
        RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_set_state_mc_moves: more than 4096 atoms per replica is not supported");
    if (n > 0 && h->cfg.system_kind == RX_SYSTEM_HARMONIC && N > 1024)
        RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_set_state_mc_moves: more than 1024 atoms per replica of a harmonic system is not supported");
    std::vector<char> seen((size_t)N);
    for (int j = 0; j < n; j++) {
        const rx_mc_move &m = moves[j];
        if (m.kind != RX_MC_DISPLACEMENT && m.kind != RX_MC_ROTATION) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: unknown move kind");
        if (!(m.sigma_nm >= 0.0) || !isfinite(m.sigma_nm)) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: sigma must be finite and >= 0");
        if (m.subset_len < 1 || m.subset_offset < 0 || (size_t)m.subset_offset + m.subset_len > h->mc_atoms.size())
            RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: subset outside the array of rx_set_mc_subsets");
        std::fill(seen.begin(), seen.end(), 0);
        const int32_t *sub = h->mc_atoms.data() + m.subset_offset;
        for (int q = 0; q < m.subset_len; q++) {
            if (seen[sub[q]]) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: a subset lists an atom twice");
            seen[sub[q]] = 1;
        }
        if (h->cfg.system_kind == RX_SYSTEM_MOLECULE) {   // every constraint cluster is in the subset wholly or not at all
            if (!h->have_particles) RX_FAIL(h, RX_ERR_INVALID, "rx_set_state_mc_moves: call rx_set_molecule first");
            for (int i = 0; i < N; i++)
                for (int q = 0; q < m.subset_len; q++)
                    if (h->mol_cluster[i] >= 0 && h->mol_cluster[i] == h->mol_cluster[sub[q]] && !seen[i])
                        RX_FAIL(h, RX_ERR_UNSUPPORTED, "rx_set_state_mc_moves: a subset holds part of a constraint cluster; a rigid "
                                                       "move keeps the constraints only when it moves whole clusters");
        }
    }
    for (int l = (state < 0 ? 0 : state); l < (state < 0 ? M : state + 1); l++)
        for (int j = 0; j < RX_MAX_MC_MOVES; j++) {
            rx_mc_move &dst = h->mc_moves[(size_t)l * RX_MAX_MC_MOVES + j];
            if (j < n) dst = moves[j];
            else { memset(&dst, 0, sizeof(dst)); dst.kind = -1; }
        }
    return upload_mc_moves(h);
}

static int mc_statistics(rx_engine *h, int64_t *acc, int64_t *prop, bool to_device, const char *who) {
    if (!acc || !prop) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": null argument");
    const size_t mm = (size_t)h->cfg.n_states * RX_MAX_MC_MOVES;
    if (!h->d_mc_acc) {
        if (to_device) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": call rx_set_mc_subsets first");
        memset(acc, 0, sizeof(int64_t) * mm);
        memset(prop, 0, sizeof(int64_t) * mm);
        return RX_OK;
    }
    if (to_device)
        for (size_t q = 0; q < mm; q++)
            if (acc[q] < 0 || prop[q] < acc[q]) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": need 0 <= accepted <= proposed");
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    const cudaMemcpyKind kind = to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
    RX_CHECK_CUDA(h, cudaMemcpy(to_device ? (void *)h->d_mc_acc : (void *)acc, to_device ? (void *)acc : (void *)h->d_mc_acc, sizeof(int64_t) * mm, kind));
    RX_CHECK_CUDA(h, cudaMemcpy(to_device ? (void *)h->d_mc_prop : (void *)prop, to_device ? (void *)prop : (void *)h->d_mc_prop, sizeof(int64_t) * mm, kind));
    return RX_OK;
}
extern "C" int rx_get_mc_statistics(rx_engine *h, int64_t *accepted, int64_t *proposed) {
    ENTER(h);
    return mc_statistics(h, accepted, proposed, false, "rx_get_mc_statistics");
}
extern "C" int rx_get_mc_energy_changes(rx_engine *h, double *du) {
    ENTER(h);
    if (!du) RX_FAIL(h, RX_ERR_INVALID, "rx_get_mc_energy_changes: null argument");
    const int K = h->cfg.n_replicas;
    for (size_t q = 0; q < (size_t)K * RX_MAX_MC_MOVES; q++) du[q] = NAN;
    if (!h->d_mc_du || h->kloc == 0) return RX_OK;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(du + (size_t)h->k0 * RX_MAX_MC_MOVES, h->d_mc_du, sizeof(double) * h->kloc * RX_MAX_MC_MOVES,
                                cudaMemcpyDeviceToHost));
    return RX_OK;
}
extern "C" int rx_set_mc_statistics(rx_engine *h, const int64_t *accepted, const int64_t *proposed) {
    ENTER(h);
    return mc_statistics(h, const_cast<int64_t *>(accepted), const_cast<int64_t *>(proposed), true, "rx_set_mc_statistics");
}

static int local_range(rx_engine *h, int first, int count, int *lo, int *n, int *skip) {
    const int K = h->cfg.n_replicas;
    if (first < 0 || count < 0 || first + count > K) RX_FAIL(h, RX_ERR_INVALID, "replica range out of bounds");
    int a = first > h->k0 ? first : h->k0;
    int b = (first + count) < (h->k0 + h->kloc) ? (first + count) : (h->k0 + h->kloc);
    if (b < a) b = a;
    *lo = a - h->k0; *n = b - a; *skip = a - first;
    return RX_OK;
}

static int set_xyz(rx_engine *h, float4 *dst, int first, int count, const double *xyz, const char *what) {
    if (h->cfg.system_kind == RX_SYSTEM_NONE) RX_FAIL(h, RX_ERR_INVALID, "engine has no particle system");
    if (!xyz) RX_FAIL(h, RX_ERR_INVALID, std::string(what) + ": null buffer");
    int lo, n, skip;
    int rc = local_range(h, first, count, &lo, &n, &skip);
    if (rc) return rc;
    return rxi_convert_in(h, dst, lo, n, xyz + (size_t)skip * h->cfg.n_atoms * 3, false);
}
static int get_xyz(rx_engine *h, const float4 *src, int first, int count, double *xyz, bool wrap, const char *what) {
    if (h->cfg.system_kind == RX_SYSTEM_NONE) RX_FAIL(h, RX_ERR_INVALID, "engine has no particle system");
    if (!xyz) RX_FAIL(h, RX_ERR_INVALID, std::string(what) + ": null buffer");
    int lo, n, skip;
    int rc = local_range(h, first, count, &lo, &n, &skip);
    if (rc) return rc;
    return rxi_convert_out(h, src, lo, n, xyz + (size_t)skip * h->cfg.n_atoms * 3, wrap);
}

extern "C" int rx_set_positions(rx_engine *h, int32_t first, int32_t count, const double *xyz) {
    ENTER(h);
    return set_xyz(h, h->d_pos, first, count, xyz, "rx_set_positions");
}
extern "C" int rx_set_velocities(rx_engine *h, int32_t first, int32_t count, const double *xyz) {
    ENTER(h);
    return set_xyz(h, h->d_vel, first, count, xyz, "rx_set_velocities");
}
extern "C" int rx_get_positions(rx_engine *h, int32_t first, int32_t count, double *xyz) {
    ENTER(h);
    // (an NPT replica's positions are left where the propagation wrapped them into its own box)
    return get_xyz(h, h->d_pos, first, count, xyz, h->cfg.system_kind == RX_SYSTEM_LJ_ALCH && !h->npt, "rx_get_positions");
}
extern "C" int rx_get_velocities(rx_engine *h, int32_t first, int32_t count, double *xyz) {
    ENTER(h);
    return get_xyz(h, h->d_vel, first, count, xyz, false, "rx_get_velocities");
}

// ---- constant pressure -------------------------------------------------------------------------------------------------
extern "C" int rx_set_pressures(rx_engine *h, const double *pressure, const double *dispersion) {
    ENTER(h);
    if (h->cfg.system_kind != RX_SYSTEM_LJ_ALCH) RX_FAIL(h, RX_ERR_INVALID, "rx_set_pressures: constant pressure needs a periodic LJ engine");
    if (!pressure || !dispersion) RX_FAIL(h, RX_ERR_INVALID, "rx_set_pressures: null argument");
    const int M = h->cfg.n_states, n = h->kloc > 0 ? h->kloc : 1;
    std::vector<double2> tab(M);
    for (int l = 0; l < M; l++) {
        if (!(pressure[l] > 0) || !isfinite(pressure[l]) || !isfinite(dispersion[l]))
            RX_FAIL(h, RX_ERR_INVALID, "rx_set_pressures: need finite pressures > 0 and finite dispersion coefficients");
        tab[l] = make_double2(pressure[l], dispersion[l]);
    }
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (!h->d_npt) {   // taken by the engine once all of them exist
        DevBuf<double2> d_npt;
        DevBuf<double4> d_box, d_box_snap;
        DevBuf<rx_barostat_state> d_baro, d_baro_snap;
        RX_CHECK_CUDA(h, d_npt.alloc(M));
        RX_CHECK_CUDA(h, d_box.alloc(n));
        RX_CHECK_CUDA(h, d_box_snap.alloc(n));
        RX_CHECK_CUDA(h, d_baro.alloc(n));
        RX_CHECK_CUDA(h, d_baro_snap.alloc(n));
        h->d_npt = std::move(d_npt); h->d_box = std::move(d_box); h->d_box_snap = std::move(d_box_snap);
        h->d_baro = std::move(d_baro); h->d_baro_snap = std::move(d_baro_snap);
    }
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_npt, tab.data(), sizeof(double2) * M, cudaMemcpyHostToDevice));
    const double *L = h->cfg.box;
    std::vector<double4> b(n, make_double4(L[0], L[1], L[2], 0.0));
    rx_barostat_state s0;
    memset(&s0, 0, sizeof(s0));
    s0.volume_scale = 0.01 * L[0] * L[1] * L[2];   // MonteCarloBarostat's initial volume scale
    std::vector<rx_barostat_state> s(n, s0);
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_box, b.data(), sizeof(double4) * n, cudaMemcpyHostToDevice));
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_baro, s.data(), sizeof(rx_barostat_state) * n, cudaMemcpyHostToDevice));
    h->npt = true;
    h->aniso = false;
    h->have_snapshot = false;   // (a snapshot without boxes cannot restore an NPT replica)
    return RX_OK;
}

extern "C" int rx_set_anisotropic_barostat(rx_engine *h, int32_t scale_mask) {
    ENTER(h);
    if (!h->npt) RX_FAIL(h, RX_ERR_INVALID, "rx_set_anisotropic_barostat: the engine has no pressure (rx_set_pressures)");
    if (scale_mask < 1 || scale_mask > 7) RX_FAIL(h, RX_ERR_INVALID, "rx_set_anisotropic_barostat: scale_mask must be 1..7");
    const int n = h->kloc > 0 ? h->kloc : 1;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (!h->d_aniso) {   // taken by the engine once both exist
        DevBuf<rx_anisotropic_barostat_state> d_aniso, d_aniso_snap;
        RX_CHECK_CUDA(h, d_aniso.alloc(n));
        RX_CHECK_CUDA(h, d_aniso_snap.alloc(n));
        h->d_aniso = std::move(d_aniso); h->d_aniso_snap = std::move(d_aniso_snap);
    }
    const double *L = h->cfg.box;
    rx_anisotropic_barostat_state s0;
    memset(&s0, 0, sizeof(s0));
    for (int d = 0; d < 3; d++) s0.volume_scale[d] = 0.01 * L[0] * L[1] * L[2];   // MonteCarloAnisotropicBarostat's start
    s0.scale_mask = scale_mask;
    std::vector<rx_anisotropic_barostat_state> s(n, s0);
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_aniso, s.data(), sizeof(rx_anisotropic_barostat_state) * n, cudaMemcpyHostToDevice));
    h->aniso = true;
    h->have_snapshot = false;   // (a snapshot without the per-axis state cannot restore the replica)
    return RX_OK;
}

// Copies between caller rows [first, first + count) and the owned replicas' rows of a per-replica device table.
template <typename T>
static int replica_rows(rx_engine *h, T *dev, int first, int count, T *host, bool to_device, const char *who) {
    if (!h->npt) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": the engine has no pressure (rx_set_pressures)");
    if (!host) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": null buffer");
    int lo, n, skip;
    int rc = local_range(h, first, count, &lo, &n, &skip);
    if (rc) return rc;
    if (n == 0) return RX_OK;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (to_device) RX_CHECK_CUDA(h, cudaMemcpy(dev + lo, host + skip, sizeof(T) * n, cudaMemcpyHostToDevice));
    else RX_CHECK_CUDA(h, cudaMemcpy(host + skip, dev + lo, sizeof(T) * n, cudaMemcpyDeviceToHost));
    return RX_OK;
}

extern "C" int rx_set_boxes(rx_engine *h, int32_t first, int32_t count, const double *edges) {
    ENTER(h);
    if (!edges || count < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_set_boxes: bad arguments");
    std::vector<double4> b((size_t)count);
    for (int i = 0; i < count; i++) {
        for (int d = 0; d < 3; d++)
            if (!(edges[3 * i + d] >= 2.0 * h->cfg.r_cutoff) || !isfinite(edges[3 * i + d]))
                RX_FAIL(h, RX_ERR_INVALID, "rx_set_boxes: every box edge must be at least twice the cutoff");
        b[i] = make_double4(edges[3 * i], edges[3 * i + 1], edges[3 * i + 2], 0.0);
    }
    return replica_rows(h, h->d_box.get(), first, count, b.data(), true, "rx_set_boxes");
}
extern "C" int rx_get_boxes(rx_engine *h, int32_t first, int32_t count, double *edges) {
    ENTER(h);
    if (!edges || count < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_get_boxes: bad arguments");
    std::vector<double4> b((size_t)count, make_double4(0.0, 0.0, 0.0, 0.0));
    int rc = replica_rows(h, h->d_box.get(), first, count, b.data(), false, "rx_get_boxes");
    if (rc) return rc;
    int lo, n, skip;
    local_range(h, first, count, &lo, &n, &skip);
    for (int i = skip; i < skip + n; i++) { edges[3 * i] = b[i].x; edges[3 * i + 1] = b[i].y; edges[3 * i + 2] = b[i].z; }
    return RX_OK;
}
extern "C" int rx_set_barostat(rx_engine *h, int32_t first, int32_t count, const rx_barostat_state *state) {
    ENTER(h);
    if (!state || count < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_set_barostat: bad arguments");
    for (int i = 0; i < count; i++)
        if (!(state[i].volume_scale > 0) || state[i].step < 0 || state[i].n_attempted < 0 || state[i].n_accepted < 0)
            RX_FAIL(h, RX_ERR_INVALID, "rx_set_barostat: need volume_scale > 0 and non-negative counters");
    return replica_rows(h, h->d_baro.get(), first, count, const_cast<rx_barostat_state *>(state), true, "rx_set_barostat");
}
extern "C" int rx_get_barostat(rx_engine *h, int32_t first, int32_t count, rx_barostat_state *state) {
    ENTER(h);
    if (!state || count < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_get_barostat: bad arguments");
    return replica_rows(h, h->d_baro.get(), first, count, state, false, "rx_get_barostat");
}
// The per-axis rows live in d_aniso; their step is the counter of d_baro, which the kernel advances.
extern "C" int rx_set_barostat_anisotropic(rx_engine *h, int32_t first, int32_t count, const rx_anisotropic_barostat_state *state) {
    ENTER(h);
    if (!state || count < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_set_barostat_anisotropic: bad arguments");
    if (!h->aniso) RX_FAIL(h, RX_ERR_INVALID, "rx_set_barostat_anisotropic: the engine has no anisotropic barostat");
    for (int i = 0; i < count; i++) {
        bool ok = state[i].step >= 0 && state[i].scale_mask >= 1 && state[i].scale_mask <= 7;
        for (int d = 0; d < 3; d++)
            ok = ok && state[i].volume_scale[d] > 0 && state[i].n_attempted[d] >= 0 && state[i].n_accepted[d] >= 0;
        if (!ok) RX_FAIL(h, RX_ERR_INVALID, "rx_set_barostat_anisotropic: need volume_scale > 0, non-negative counters and a mask of 1..7");
    }
    std::vector<rx_barostat_state> b((size_t)count);
    int rc = replica_rows(h, h->d_baro.get(), first, count, b.data(), false, "rx_set_barostat_anisotropic");
    if (rc) return rc;
    for (int i = 0; i < count; i++) b[i].step = state[i].step;
    rc = replica_rows(h, h->d_aniso.get(), first, count, const_cast<rx_anisotropic_barostat_state *>(state), true,
                      "rx_set_barostat_anisotropic");
    if (rc) return rc;
    return replica_rows(h, h->d_baro.get(), first, count, b.data(), true, "rx_set_barostat_anisotropic");
}
extern "C" int rx_get_barostat_anisotropic(rx_engine *h, int32_t first, int32_t count, rx_anisotropic_barostat_state *state) {
    ENTER(h);
    if (!state || count < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_get_barostat_anisotropic: bad arguments");
    if (!h->aniso) RX_FAIL(h, RX_ERR_INVALID, "rx_get_barostat_anisotropic: the engine has no anisotropic barostat");
    std::vector<rx_barostat_state> b((size_t)count);
    int rc = replica_rows(h, h->d_baro.get(), first, count, b.data(), false, "rx_get_barostat_anisotropic");
    if (rc) return rc;
    rc = replica_rows(h, h->d_aniso.get(), first, count, state, false, "rx_get_barostat_anisotropic");
    if (rc) return rc;
    int lo, n, skip;
    local_range(h, first, count, &lo, &n, &skip);
    for (int i = skip; i < skip + n; i++) state[i].step = b[i].step;
    return RX_OK;
}

bool rxi_is_pinned(const rx_engine *h, const void *p, size_t bytes) {
    const char *c = (const char *)p;
    for (const auto &r : h->pinned)
        if (c >= r.first && c + bytes <= r.first + r.second) return true;
    return false;
}

/* Page-lock a caller buffer (cudaHostRegister) so that rx_set_* / rx_get_* copy straight between it and the device instead
 * of staging through the engine's own pinned buffer: the host-resident SamplerStates of MultiStateSampler live in one
 * such buffer.  The engine unregisters what is still registered when it is destroyed. */
extern "C" int rx_pin_host_memory(rx_engine *h, void *ptr, uint64_t bytes) {
    ENTER(h);
    if (!ptr || !bytes) RX_FAIL(h, RX_ERR_INVALID, "rx_pin_host_memory: null buffer");
    RX_CHECK_CUDA(h, cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterDefault));
    h->pinned.push_back(std::make_pair((const char *)ptr, (size_t)bytes));
    return RX_OK;
}
extern "C" int rx_unpin_host_memory(rx_engine *h, void *ptr) {
    ENTER(h);
    for (size_t q = 0; q < h->pinned.size(); q++)
        if (h->pinned[q].first == (const char *)ptr) {
            RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
            cudaHostUnregister(ptr);
            h->pinned.erase(h->pinned.begin() + q);
            return RX_OK;
        }
    RX_FAIL(h, RX_ERR_INVALID, "rx_unpin_host_memory: buffer was not registered");
}

extern "C" int rx_get_replica_energies(rx_engine *h, double *potential, double *kinetic) {
    ENTER(h);
    const int K = h->cfg.n_replicas;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (potential) RX_CHECK_CUDA(h, cudaMemcpy(potential, h->d_pot, sizeof(double) * K, cudaMemcpyDeviceToHost));
    if (kinetic) RX_CHECK_CUDA(h, cudaMemcpy(kinetic, h->d_kin, sizeof(double) * K, cudaMemcpyDeviceToHost));
    return RX_OK;
}

extern "C" int rx_randomize_velocities(rx_engine *h, uint64_t seed, uint64_t stream) {
    ENTER(h);
    if (!h->have_particles || !h->have_states) RX_FAIL(h, RX_ERR_INVALID, "rx_randomize_velocities: set particles and states first");
    return rxi_randomize_velocities(h, seed, stream);
}

extern "C" int rx_minimize(rx_engine *h, double tolerance, int32_t max_iterations, double *rms_force, int32_t *iterations) {
    ENTER(h);
    if (!h->have_particles || !h->have_states) RX_FAIL(h, RX_ERR_INVALID, "rx_minimize: set particles and states first");
    if (!(tolerance > 0.0)) RX_FAIL(h, RX_ERR_INVALID, "rx_minimize: tolerance must be positive");
    if (max_iterations < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_minimize: max_iterations must be >= 0");
    const int K = h->cfg.n_replicas;
    DevBuf<double> d_rms;
    DevBuf<int> d_it;
    RX_CHECK_CUDA(h, d_rms.alloc(K));
    RX_CHECK_CUDA(h, d_it.alloc(K));
    cudaMemsetAsync(d_rms, 0, sizeof(double) * K, h->stream);
    cudaMemsetAsync(d_it, 0, sizeof(int) * K, h->stream);
    int rc = rxi_minimize(h, tolerance, max_iterations == 0 ? 20000 : max_iterations, d_rms, d_it);
    if (rc == RX_OK && cudaStreamSynchronize(h->stream) != cudaSuccess) { h->err = "rx_minimize: kernel failed"; rc = RX_ERR_CUDA; }
    if (rc == RX_OK && rms_force) cudaMemcpy(rms_force, d_rms, sizeof(double) * K, cudaMemcpyDeviceToHost);
    if (rc == RX_OK && iterations) cudaMemcpy(iterations, d_it, sizeof(int) * K, cudaMemcpyDeviceToHost);
    return rc;
}

extern "C" int rx_set_replica_states(rx_engine *h, const int64_t *states) {
    ENTER(h);
    const int K = h->cfg.n_replicas, M = h->cfg.n_states;
    std::vector<int> p(K);
    for (int k = 0; k < K; k++) {
        if (states[k] < 0 || states[k] >= M) RX_FAIL(h, RX_ERR_INVALID, "rx_set_replica_states: state index out of range");
        p[k] = (int)states[k];
    }
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_perm, p.data(), sizeof(int) * K, cudaMemcpyHostToDevice));
    return RX_OK;
}
extern "C" int rx_get_replica_states(rx_engine *h, int64_t *states) {
    ENTER(h);
    const int K = h->cfg.n_replicas;
    std::vector<int> p(K);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(p.data(), h->d_perm, sizeof(int) * K, cudaMemcpyDeviceToHost));
    for (int k = 0; k < K; k++) states[k] = p[k];
    return RX_OK;
}

static int check_ready(rx_engine *h, const char *who) {
    if (h->cfg.system_kind == RX_SYSTEM_NONE) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": engine has no particle system");
    if (!h->have_particles || !h->have_states) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": rx_set_particles and rx_set_states must be called first");
    return RX_OK;
}

static int check_device_error(rx_engine *h) {
    int e = 0;
    RX_CHECK_CUDA(h, cudaMemcpy(&e, h->d_err, sizeof(int), cudaMemcpyDeviceToHost));
    if (e) {
        cudaMemset(h->d_err, 0, sizeof(int));
        RX_FAIL(h, e, e == RX_ERR_CAPACITY ? "lambda-controlled pair list overflowed its capacity" : "device-side error");
    }
    return RX_OK;
}

static int finish_propagate(rx_engine *h, PhaseTimer &T, int32_t *nan_flags, const char *who);

extern "C" int rx_propagate(rx_engine *h, uint64_t seed, uint64_t iteration, int32_t reassign, int32_t *nan_flags) {
    ENTER(h);
    int rc = check_ready(h, "rx_propagate");
    if (rc) return rc;
    if (!h->have_integrator) RX_FAIL(h, RX_ERR_INVALID, "rx_propagate: rx_set_integrator must be called first");
    PhaseTimer T(h, 1);
    int launches = 0;
    rc = rxi_mc_moves(h, seed, iteration, &launches);   // (before the snapshot: a retry reruns the dynamics only)
    if (rc) return rc;
    rc = rxi_snapshot_state(h);
    if (rc) return rc;
    rc = rxi_propagate(h, seed, iteration, reassign, &launches);
    if (rc) return rc;
    T.stop(launches);
    return finish_propagate(h, T, nan_flags, "rx_propagate");
}

/* Replaces the restart loop of BaseIntegratorMove.apply (openmmtools/mcmc.py:706-759): the replicas whose NaN flag is set
 * go back to the state they had when rx_propagate began and are propagated again (other noise: pass another seed); the
 * replicas that came through are left alone. */
extern "C" int rx_propagate_retry(rx_engine *h, uint64_t seed, uint64_t iteration, int32_t reassign, int32_t *nan_flags) {
    ENTER(h);
    int rc = check_ready(h, "rx_propagate_retry");
    if (rc) return rc;
    if (!h->have_integrator) RX_FAIL(h, RX_ERR_INVALID, "rx_propagate_retry: rx_set_integrator must be called first");
    PhaseTimer T(h, 1);
    int launches = 0;
    rc = rxi_restore_failed(h);
    if (rc) return rc;
    rc = rxi_propagate(h, seed, iteration, reassign, &launches, h->d_retry);
    if (rc) return rc;
    T.stop(launches + 1);
    return finish_propagate(h, T, nan_flags, "rx_propagate_retry");
}

static int finish_propagate(rx_engine *h, PhaseTimer &T, int32_t *nan_flags, const char *who) {
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    T.accumulate();
    const int K = h->cfg.n_replicas;
    std::vector<int> f(K, 0);
    RX_CHECK_CUDA(h, cudaMemcpy(f.data(), h->d_nan, sizeof(int) * K, cudaMemcpyDeviceToHost));
    int any = 0;
    for (int k = 0; k < K; k++) {
        const bool mine = k >= h->k0 && k < h->k0 + h->kloc;
        const int v = mine ? f[k] : 0;
        if (nan_flags) nan_flags[k] = v;
        any |= v;
    }
    if (any) RX_FAIL(h, RX_ERR_NAN, std::string(who) + ": NaN encountered in positions, velocities or potential energy");
    return RX_OK;
}

extern "C" int rx_compute_energies(rx_engine *h, double *u_out) {
    ENTER(h);
    int rc = check_ready(h, "rx_compute_energies");
    if (rc) return rc;
    PhaseTimer T(h, 2);
    int launches = 0;
    rc = rxi_compute_energy_rows(h, &launches);
    if (rc) return rc;
    rc = rxi_allgather_energies(h);
    if (rc) return rc;
    T.stop(launches);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    T.accumulate();
    rc = check_device_error(h);
    if (rc) return rc;
    if (u_out) RX_CHECK_CUDA(h, cudaMemcpy(u_out, h->d_u, sizeof(double) * (size_t)h->cfg.n_replicas * h->cfg.n_states, cudaMemcpyDeviceToHost));
    return RX_OK;
}

extern "C" int rx_set_energies(rx_engine *h, const double *u) {
    ENTER(h);
    if (!u) RX_FAIL(h, RX_ERR_INVALID, "rx_set_energies: null");
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(h->d_u, u, sizeof(double) * (size_t)h->cfg.n_replicas * h->cfg.n_states, cudaMemcpyHostToDevice));
    return RX_OK;
}
extern "C" int rx_get_energies(rx_engine *h, double *u) {
    ENTER(h);
    if (!u) RX_FAIL(h, RX_ERR_INVALID, "rx_get_energies: null");
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    RX_CHECK_CUDA(h, cudaMemcpy(u, h->d_u, sizeof(double) * (size_t)h->cfg.n_replicas * h->cfg.n_states, cudaMemcpyDeviceToHost));
    return RX_OK;
}

// Energies at n other states; pressure / dispersion (NPT engines only, else NULL) are those states' (p, c) tables.
// lambda2 (NULL: 1) is those states' lambda of the second alchemical region.
static int energies_at(rx_engine *h, const rx_state_params *st, const double *lambda2, const double *pressure,
                       const double *dispersion, int32_t n, double *u_out, const char *who) {
    int rc = check_ready(h, who);
    if (rc) return rc;
    if (!st || !u_out || n < 1) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": bad arguments");
    std::vector<StateDev> hs;
    rc = convert_states(h, st, n, hs, who);
    if (!rc) rc = convert_states_region2(h, lambda2, n, hs, who);
    if (rc) return rc;
    std::vector<double2> tab;
    if (pressure) {
        for (int l = 0; l < n; l++) {
            if (!(pressure[l] > 0) || !isfinite(pressure[l]) || !isfinite(dispersion[l]))
                RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": need finite pressures > 0 and finite dispersion coefficients");
            tab.push_back(make_double2(pressure[l], dispersion[l]));
        }
    }
    const int K = h->cfg.n_replicas;
    DevBuf<StateDev> d_st;
    DevBuf<double2> d_tab;
    RX_CHECK_CUDA(h, d_st.alloc(n));
    // the result stays in d_u_at, where rx_history_append finds the unsampled block
    h->u_at_cols = 0;
    if ((size_t)K * n > h->u_at_cap) {
        RX_CHECK_CUDA(h, h->d_u_at.alloc((size_t)K * n));
        h->u_at_cap = (size_t)K * n;
    }
    double *d_out = h->d_u_at;
    if (pressure) RX_CHECK_CUDA(h, d_tab.alloc(n));
    int launches = 0;
    cudaMemcpyAsync(d_st, hs.data(), sizeof(StateDev) * n, cudaMemcpyHostToDevice, h->stream);
    if (pressure) cudaMemcpyAsync(d_tab, tab.data(), sizeof(double2) * n, cudaMemcpyHostToDevice, h->stream);
    cudaMemsetAsync(d_out, 0, sizeof(double) * (size_t)K * n, h->stream);
    rc = rxi_compute_energy_rows_at(h, d_st, n, d_out, &launches, d_tab);
    if (!rc) rc = rxi_allgather_rows(h, d_out, n);
    if (!rc) {
        cudaError_t e = cudaMemcpyAsync(u_out, d_out, sizeof(double) * (size_t)K * n, cudaMemcpyDeviceToHost, h->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
        if (e != cudaSuccess) { h->err = std::string(who) + ": " + cudaGetErrorString(e); rc = RX_ERR_CUDA; }
    }
    cudaStreamSynchronize(h->stream);   // (before the buffers are freed)
    if (rc) return rc;
    h->phase_launches[2] += launches;
    rc = check_device_error(h);
    if (!rc) h->u_at_cols = n;
    return rc;
}

// ---- energy history -------------------------------------------------------------------------------------------------
// Capacity for `rows` rows of M + U doubles per replica, grown geometrically.  The growth is checked against the free
// device memory first, and a growth that fails leaves the history as it was.
static int history_reserve(rx_engine *h, long long rows, int U, const char *who) {
    const size_t row = (size_t)h->cfg.n_replicas * (h->cfg.n_states + U);
    if (rows < 0 || U < 0) RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": negative size");
    if (h->hist_len > 0 && U != h->hist_u)
        RX_FAIL(h, RX_ERR_INVALID, std::string(who) + ": the history holds " + std::to_string(h->hist_u) + " unsampled states");
    if ((size_t)rows * row <= h->hist_cap) return RX_OK;
    const size_t want = std::max((size_t)rows * row, std::max((size_t)16 * row, 2 * h->hist_cap));
    size_t free_b = 0, total_b = 0;
    RX_CHECK_CUDA(h, cudaMemGetInfo(&free_b, &total_b));
    if (rows > (long long)(SIZE_MAX / 16 / row) || want * sizeof(double) > free_b)
        RX_FAIL(h, RX_ERR_UNSUPPORTED, std::string(who) + ": an energy history of " + std::to_string(rows) +
                                           " iterations needs " + std::to_string(want * sizeof(double)) + " bytes, the device has " +
                                           std::to_string(free_b) + " free");
    DevBuf<double> grown;
    const cudaError_t e = grown.alloc(want);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        RX_FAIL(h, RX_ERR_UNSUPPORTED, std::string(who) + ": out of device memory for the energy history");
    }
    RX_CHECK_CUDA(h, e);
    if (h->hist_len > 0)
        RX_CHECK_CUDA(h, cudaMemcpyAsync(grown, h->d_hist, (size_t)h->hist_len * row * sizeof(double), cudaMemcpyDeviceToDevice,
                                         h->stream));
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    h->d_hist = std::move(grown);
    h->hist_cap = want;
    return RX_OK;
}

extern "C" int rx_history_reserve(rx_engine *h, int64_t n_iterations, int32_t n_unsampled) {
    ENTER(h);
    return history_reserve(h, n_iterations, n_unsampled, "rx_history_reserve");
}

extern "C" int rx_history_append(rx_engine *h, int64_t iteration, int32_t n_unsampled) {
    ENTER(h);
    if (iteration < 0 || iteration > h->hist_len)
        RX_FAIL(h, RX_ERR_INVALID, "rx_history_append: iteration " + std::to_string(iteration) + " does not follow the " +
                                       std::to_string(h->hist_len) + " iterations of the history");
    if (n_unsampled > 0 && h->u_at_cols != n_unsampled)
        RX_FAIL(h, RX_ERR_INVALID, "rx_history_append: the last rx_compute_energies_at call did not compute " +
                                       std::to_string(n_unsampled) + " states");
    const long long len = h->hist_len;
    if (iteration == 0) h->hist_len = 0;    // a new history may change the number of unsampled states
    int rc = history_reserve(h, iteration + 1, n_unsampled, "rx_history_append");
    if (rc) { h->hist_len = len; return rc; }
    const int K = h->cfg.n_replicas, M = h->cfg.n_states, W = M + n_unsampled;
    double *row = h->d_hist + (size_t)iteration * K * W;
    RX_CHECK_CUDA(h, cudaMemcpy2DAsync(row, W * sizeof(double), h->d_u, M * sizeof(double), M * sizeof(double), K,
                                       cudaMemcpyDeviceToDevice, h->stream));
    if (n_unsampled > 0)
        RX_CHECK_CUDA(h, cudaMemcpy2DAsync(row + M, W * sizeof(double), h->d_u_at, n_unsampled * sizeof(double),
                                           n_unsampled * sizeof(double), K, cudaMemcpyDeviceToDevice, h->stream));
    h->hist_len = iteration + 1;
    h->hist_u = n_unsampled;
    return RX_OK;
}

extern "C" int rx_history_truncate(rx_engine *h, int64_t iteration) {
    ENTER(h);
    if (iteration < -1) RX_FAIL(h, RX_ERR_INVALID, "rx_history_truncate: iteration must be >= -1");
    h->hist_len = std::min(h->hist_len, (long long)iteration + 1);
    return RX_OK;
}

extern "C" int rx_history_load(rx_engine *h, int64_t n_iterations, int32_t n_unsampled, const double *u,
                               const double *u_unsampled) {
    ENTER(h);
    if (n_iterations < 0 || n_unsampled < 0 || (n_iterations > 0 && !u) || (n_iterations > 0 && n_unsampled > 0 && !u_unsampled))
        RX_FAIL(h, RX_ERR_INVALID, "rx_history_load: bad arguments");
    const long long len = h->hist_len;
    h->hist_len = 0;     // (the old rows are not kept)
    int rc = history_reserve(h, n_iterations, n_unsampled, "rx_history_load");
    if (rc) { h->hist_len = len; return rc; }
    const int M = h->cfg.n_states, W = M + n_unsampled;
    const size_t height = (size_t)n_iterations * h->cfg.n_replicas;
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    if (height > 0) {
        RX_CHECK_CUDA(h, cudaMemcpy2D(h->d_hist, W * sizeof(double), u, M * sizeof(double), M * sizeof(double), height,
                                      cudaMemcpyHostToDevice));
        if (n_unsampled > 0)
            RX_CHECK_CUDA(h, cudaMemcpy2D(h->d_hist + M, W * sizeof(double), u_unsampled, n_unsampled * sizeof(double),
                                          n_unsampled * sizeof(double), height, cudaMemcpyHostToDevice));
    }
    h->hist_len = n_iterations;
    h->hist_u = n_unsampled;
    return RX_OK;
}

extern "C" int rx_history_length(rx_engine *h, int64_t *n_iterations, int32_t *n_unsampled) {
    ENTER(h);
    if (n_iterations) *n_iterations = h->hist_len;
    if (n_unsampled) *n_unsampled = h->hist_u;
    return RX_OK;
}

extern "C" int rx_compute_energies_at(rx_engine *h, const rx_state_params *st, int32_t n, double *u_out) {
    ENTER(h);
    return energies_at(h, st, nullptr, nullptr, nullptr, n, u_out, "rx_compute_energies_at");
}

extern "C" int rx_compute_energies_at_npt(rx_engine *h, const rx_state_params *st, const double *pressure,
                                          const double *dispersion, int32_t n, double *u_out) {
    ENTER(h);
    if (!pressure || !dispersion) RX_FAIL(h, RX_ERR_INVALID, "rx_compute_energies_at_npt: null argument");
    return energies_at(h, st, nullptr, pressure, dispersion, n, u_out, "rx_compute_energies_at_npt");
}

extern "C" int rx_compute_energies_at_region2(rx_engine *h, const rx_state_params *st, const double *lambda2,
                                              const double *pressure, const double *dispersion, int32_t n, double *u_out) {
    ENTER(h);
    if (!lambda2 || (!pressure) != (!dispersion)) RX_FAIL(h, RX_ERR_INVALID, "rx_compute_energies_at_region2: null argument");
    return energies_at(h, st, lambda2, pressure, dispersion, n, u_out, "rx_compute_energies_at_region2");
}

extern "C" int rx_mix_seed(rx_engine *h, int32_t stream, uint32_t seed) {
    ENTER(h);
    return rxi_mix_seed(h, stream, seed);
}
extern "C" int rx_mix_skip(rx_engine *h, int32_t stream, uint64_t n_words) {
    ENTER(h);
    return rxi_mix_skip(h, stream, n_words);
}

static int fetch_mix_results(rx_engine *h, int64_t *states_out, int64_t *nacc, int64_t *nprop) {
    const size_t mm = (size_t)h->cfg.n_states * h->cfg.n_states;
    if (states_out) { int rc = rx_get_replica_states(h, states_out); if (rc) return rc; }
    if (nacc) RX_CHECK_CUDA(h, cudaMemcpy(nacc, h->d_nacc, sizeof(int64_t) * mm, cudaMemcpyDeviceToHost));
    if (nprop) RX_CHECK_CUDA(h, cudaMemcpy(nprop, h->d_nprop, sizeof(int64_t) * mm, cudaMemcpyDeviceToHost));
    return RX_OK;
}

extern "C" int rx_mix_swap_all(rx_engine *h, int64_t nswap, int64_t *states_out, int64_t *nacc, int64_t *nprop) {
    ENTER(h);
    if (nswap < 0) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_swap_all: nswap_attempts must be >= 0");
    PhaseTimer T(h, 0);
    int launches = 0;
    int rc = rxi_mix_swap_all(h, nswap, &launches);
    if (rc) return rc;
    T.stop(launches);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    T.accumulate();
    return fetch_mix_results(h, states_out, nacc, nprop);
}

extern "C" int rx_mix_swap_neighbors(rx_engine *h, int64_t *states_out, int64_t *nacc, int64_t *nprop) {
    ENTER(h);
    PhaseTimer T(h, 0);
    int launches = 0;
    int rc = rxi_mix_swap_neighbors(h, &launches);
    if (rc) return rc;
    T.stop(launches);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    T.accumulate();
    return fetch_mix_results(h, states_out, nacc, nprop);
}

extern "C" int rx_get_mix_counts(rx_engine *h, int64_t *nacc, int64_t *nprop) {
    ENTER(h);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    return fetch_mix_results(h, nullptr, nacc, nprop);
}

extern "C" int rx_mix_stream_position(rx_engine *h, int32_t stream, uint64_t *words) {
    ENTER(h);
    if (stream < 0 || stream > 1 || !words) RX_FAIL(h, RX_ERR_INVALID, "rx_mix_stream_position: bad arguments");
    *words = h->streams[stream].consumed;
    return RX_OK;
}

// The fused loop of rx_run_iterations and rx_sams_run_iterations, multistatesampler.py:776-782 without a host round trip:
// mix (with the previous iteration's energies) -> propagate -> energies.  mix(iteration, &launches) is the mixing step; `who`
// names the entry point in errors.
template <class Mix>
static int run_fused(rx_engine *h, const char *who, int32_t n_iterations, uint64_t seed, uint64_t first_iteration, int32_t reassign,
                     Mix mix) {
    int rc;
    for (int it = 0; it < n_iterations; it++) {
        int lm = 0, lp = 0, le = 0;
        PhaseTimer Tm(h, 0);
        rc = mix(first_iteration + it, &lm);
        if (rc) return rc;
        Tm.stop(lm);
        PhaseTimer Tp(h, 1);
        rc = rxi_mc_moves(h, seed, first_iteration + it, &lp);
        if (rc) return rc;
        rc = rxi_propagate(h, seed, first_iteration + it, reassign, &lp);
        if (rc) return rc;
        Tp.stop(lp);
        PhaseTimer Te(h, 2);
        rc = rxi_compute_energy_rows(h, &le);
        if (rc) return rc;
        rc = rxi_allgather_energies(h);
        if (rc) return rc;
        Te.stop(le);
        RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
        Tm.accumulate(); Tp.accumulate(); Te.accumulate();
    }
    rc = check_device_error(h);
    if (rc) return rc;
    std::vector<int> f(h->cfg.n_replicas, 0);
    RX_CHECK_CUDA(h, cudaMemcpy(f.data(), h->d_nan, sizeof(int) * f.size(), cudaMemcpyDeviceToHost));
    for (int k = h->k0; k < h->k0 + h->kloc; k++)
        if (f[k]) RX_FAIL(h, RX_ERR_NAN, std::string(who) + ": NaN encountered in a replica");
    return RX_OK;
}

extern "C" int rx_run_iterations(rx_engine *h, int32_t n_iterations, int32_t mixing, uint64_t seed,
                                 uint64_t first_iteration, int32_t reassign) {
    ENTER(h);
    int rc = check_ready(h, "rx_run_iterations");
    if (rc) return rc;
    if (!h->have_integrator) RX_FAIL(h, RX_ERR_INVALID, "rx_run_iterations: rx_set_integrator must be called first");
    if (mixing < 0 || mixing > 2) RX_FAIL(h, RX_ERR_INVALID, "rx_run_iterations: mixing must be 0, 1 or 2");
    const long long K = h->cfg.n_replicas;
    return run_fused(h, "rx_run_iterations", n_iterations, seed, first_iteration, reassign, [&](uint64_t, int *lm) {
        if (mixing == 1) return rxi_mix_swap_all(h, K * K * K, lm);
        if (mixing == 2) return rxi_mix_swap_neighbors(h, lm);
        return (int)RX_OK;
    });
}

// ---- SAMS (rx_sams.cuh) ------------------------------------------------------------------------------------------------------
extern "C" int rx_sams_set(rx_engine *h, const rx_sams_config *config, const double *log_target, const double *logZ,
                           const int64_t *histogram) {
    ENTER(h);
    if (!config || !log_target || !logZ) RX_FAIL(h, RX_ERR_INVALID, "rx_sams_set: null argument");
    return rxi_sams_set(h, config, log_target, logZ, histogram);
}

extern "C" int rx_sams_step(rx_engine *h, int64_t iteration, int32_t update_weights, const int64_t *histogram) {
    ENTER(h);
    int rc = check_ready(h, "rx_sams_step");
    if (rc) return rc;
    if (histogram && (rc = rxi_sams_set_histogram(h, histogram))) return rc;
    int lm = 0;
    PhaseTimer Tm(h, 0);
    rc = rxi_sams_step(h, iteration, update_weights, &lm);
    if (rc) return rc;
    Tm.stop(lm);
    RX_CHECK_CUDA(h, cudaStreamSynchronize(h->stream));
    Tm.accumulate();
    return check_device_error(h);
}

extern "C" int rx_sams_get(rx_engine *h, double *logZ, double *log_weights, int64_t *histogram, int32_t *stage, int64_t *t0,
                           double *gamma, int64_t *states, int64_t *previous_states) {
    ENTER(h);
    return rxi_sams_get(h, logZ, log_weights, histogram, stage, t0, gamma, states, previous_states);
}

extern "C" int rx_sams_run_iterations(rx_engine *h, int32_t n_iterations, uint64_t seed, uint64_t first_iteration, int32_t reassign) {
    ENTER(h);
    int rc = check_ready(h, "rx_sams_run_iterations");
    if (rc) return rc;
    if (!h->have_integrator) RX_FAIL(h, RX_ERR_INVALID, "rx_sams_run_iterations: rx_set_integrator must be called first");
    // sams.py:395-437 as the mixing: jump + weight update
    return run_fused(h, "rx_sams_run_iterations", n_iterations, seed, first_iteration, reassign, [&](uint64_t iteration, int *lm) {
        return rxi_sams_step(h, (long long)iteration, iteration > 0 ? 1 : 0, lm);
    });
}

extern "C" int rx_get_phase_times(rx_engine *h, double ms[4], int64_t counts[4], int32_t reset) {
    ENTER(h);
    for (int i = 0; i < 4; i++) {
        if (ms) ms[i] = h->phase_ms[i];
        if (counts) counts[i] = h->phase_launches[i];
        if (reset) { h->phase_ms[i] = 0; h->phase_launches[i] = 0; }
    }
    return RX_OK;
}

extern "C" int rx_timer_mark(rx_engine *h, int32_t which) {
    ENTER(h);
    if (which < 0 || which > 1) RX_FAIL(h, RX_ERR_INVALID, "rx_timer_mark: which must be 0 or 1");
    RX_CHECK_CUDA(h, cudaEventRecord(h->ev_user[which], h->stream));
    return RX_OK;
}
extern "C" int rx_timer_elapsed(rx_engine *h, double *ms) {
    ENTER(h);
    if (!ms) RX_FAIL(h, RX_ERR_INVALID, "rx_timer_elapsed: null");
    RX_CHECK_CUDA(h, cudaEventSynchronize(h->ev_user[1]));
    float f = 0;
    RX_CHECK_CUDA(h, cudaEventElapsedTime(&f, h->ev_user[0], h->ev_user[1]));
    *ms = f;
    return RX_OK;
}
extern "C" int rx_selftest_exp(rx_engine *h, const double *x, double *y, int32_t n) {
    if (!h) return RX_ERR_INVALID;
    if (n > 0 && (!x || !y)) RX_FAIL(h, RX_ERR_INVALID, "rx_selftest_exp: null array");
    RX_CHECK_CUDA(h, cudaSetDevice(h->cfg.device));
    return rxi_selftest_exp(h, x, y, n);
}
extern "C" int rx_plan_propagate(const rx_propagate_query *q, rx_propagate_plan *out) {
    if (!q || !out) { g_rx_create_error = "rx_plan_propagate: null argument"; return RX_ERR_INVALID; }
    return rxi_plan_propagate(q, out, g_rx_create_error);
}

extern "C" int rx_get_mix_stats(rx_engine *h, int64_t out[6]) {
    ENTER(h);
    for (int i = 0; i < 6; i++) out[i] = h->mix_stats[i];
    return RX_OK;
}

// ---- NCCL through dlopen: the single-GPU path has no NCCL dependency -------------------------------
typedef struct { char internal[128]; } rx_nccl_id;
typedef int (*nccl_get_id_t)(rx_nccl_id *);
typedef int (*nccl_init_rank_t)(void **, int, rx_nccl_id, int);
typedef int (*nccl_allgather_t)(const void *, void *, size_t, int, void *, cudaStream_t);
typedef const char *(*nccl_errstr_t)(int);
#define RX_NCCL_FLOAT64 8 /* ncclFloat64 / ncclDouble in nccl.h's ncclDataType_t */

extern "C" int rx_comm_unique_id(const char *path, void *id_out) {
    if (!path || !id_out) { g_rx_create_error = "rx_comm_unique_id: null argument"; return RX_ERR_INVALID; }
    void *lib = dlopen(path, RTLD_NOW | RTLD_GLOBAL);
    if (!lib) { g_rx_create_error = std::string("dlopen failed: ") + dlerror(); return RX_ERR_COMM; }
    nccl_get_id_t f = (nccl_get_id_t)dlsym(lib, "ncclGetUniqueId");
    if (!f) { g_rx_create_error = "ncclGetUniqueId not found"; return RX_ERR_COMM; }
    rx_nccl_id id;
    int r = f(&id);
    if (r != 0) { g_rx_create_error = "ncclGetUniqueId failed"; return RX_ERR_COMM; }
    memcpy(id_out, &id, sizeof(id));
    return RX_OK;
}

extern "C" int rx_comm_init(rx_engine *h, const char *path, const void *unique_id) {
    ENTER(h);
    if (h->cfg.world_size == 1) return RX_OK;
    if (!path || !unique_id) RX_FAIL(h, RX_ERR_INVALID, "rx_comm_init: null argument");
    h->nccl_lib = dlopen(path, RTLD_NOW | RTLD_GLOBAL);
    if (!h->nccl_lib) RX_FAIL(h, RX_ERR_COMM, std::string("dlopen failed: ") + dlerror());
    nccl_init_rank_t f = (nccl_init_rank_t)dlsym(h->nccl_lib, "ncclCommInitRank");
    if (!f) RX_FAIL(h, RX_ERR_COMM, "ncclCommInitRank not found");
    rx_nccl_id id;
    memcpy(&id, unique_id, sizeof(id));
    int r = f(&h->nccl_comm, h->cfg.world_size, id, h->cfg.rank);
    if (r != 0) {
        nccl_errstr_t es = (nccl_errstr_t)dlsym(h->nccl_lib, "ncclGetErrorString");
        RX_FAIL(h, RX_ERR_COMM, std::string("ncclCommInitRank failed: ") + (es ? es(r) : "?"));
    }
    if ((h->cfg.n_replicas % h->cfg.world_size) != 0) RX_FAIL(h, RX_ERR_INVALID, "rx_comm_init: n_replicas must be divisible by world_size");
    return RX_OK;
}

int rxi_allgather_rows(rx_engine *h, double *d_matrix, int n_cols) {
    if (h->cfg.world_size == 1) return RX_OK;
    if (!h->nccl_comm) RX_FAIL(h, RX_ERR_COMM, "world_size > 1 but rx_comm_init has not been called");
    nccl_allgather_t f = (nccl_allgather_t)dlsym(h->nccl_lib, "ncclAllGather");
    if (!f) RX_FAIL(h, RX_ERR_COMM, "ncclAllGather not found");
    const size_t cnt = (size_t)h->kloc * n_cols;
    // in place: each rank's rows already sit at their final offset
    int r = f(d_matrix + (size_t)h->k0 * n_cols, d_matrix, cnt, RX_NCCL_FLOAT64, h->nccl_comm, h->stream);
    if (r != 0) RX_FAIL(h, RX_ERR_COMM, "ncclAllGather failed");
    return RX_OK;
}

int rxi_allgather_energies(rx_engine *h) { return rxi_allgather_rows(h, h->d_u, h->cfg.n_states); }
