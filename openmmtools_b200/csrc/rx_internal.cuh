// rx_internal.cuh -- shared declarations of librx_b200.so (not part of the public ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <memory>
#include <string>
#include <vector>
#include <utility>
#include "../../include/rx_b200.h"

#define RX_KB 8.31446261815324e-3 /* kJ/mol/K, openmmtools/constants.py:7 with OpenMM >= 7.6 CODATA-2018 values */
#define RX_MAX_PROGRAM 32

// ---- per-state table as the kernels see it ---------------------------------------------------------
struct StateDev {
    double beta;     // 1/(kB T)
    double kT;       // kB T
    double lambda;   // lambda_sterics
    double la;       // lambda^a            (alchemy.py:1385)
    double ob;       // alpha (1-lambda)^b  (alchemy.py:1388)
    double offset;   // kJ/mol
    double ho_K;
    double ho_x0[3];
    // the second alchemical region's lambda_sterics<suffix> and its two soft-core factors (rx_set_states_region2);
    // read only by the two-region kernels
    double lambda2, la2, ob2;
    // lambda_electrostatics (rx_state_params); read only by the alchemical molecule kernels
    double lambda_e;
};

// ---- owned memory ---------------------------------------------------------------------------------------------------
// n elements of T in device memory (Pinned: page-locked host memory), freed by the destructor.  Move-only.  It converts to its
// raw pointer: the kernels' arguments and parameter structs (MolDev, MolGB, EnParams, DynParams) are views of owned memory.
template <typename T, bool Pinned = false> class CudaBuf {
  public:
    CudaBuf() = default;
    CudaBuf(CudaBuf &&o) noexcept : p_(o.p_) { o.p_ = nullptr; }
    CudaBuf &operator=(CudaBuf &&o) noexcept {
        if (this != &o) { release(p_); p_ = o.p_; o.p_ = nullptr; }
        return *this;
    }
    ~CudaBuf() { release(p_); }
    operator T *() const { return p_; }
    T *get() const { return p_; }
    // n elements of `elem` bytes each in place of what it holds, which is released only once the new storage exists: a
    // failure leaves the buffer as it was.
    cudaError_t alloc(size_t n, size_t elem = sizeof(T)) {
        void *q = nullptr;
        const cudaError_t e = Pinned ? cudaHostAlloc(&q, n * elem, cudaHostAllocDefault) : cudaMalloc(&q, n * elem);
        if (e == cudaSuccess) { release(p_); p_ = (T *)q; }
        return e;
    }

  private:
    static void release(T *p) { if (p && Pinned) cudaFreeHost(p); else if (p) cudaFree(p); }
    T *p_ = nullptr;
};
template <typename T> using DevBuf = CudaBuf<T>;
template <typename T> using PinnedBuf = CudaBuf<T, true>;

struct MoveDev;     // rx_dynamics.cu: the elements of rx_engine::d_moves
// Host records that own device buffers, complete only in the translation unit that uses them, where each overload of
// RecordDelete is defined.
struct SamsState;   // rx_sams.cuh
struct MolTables;   // rx_dynamics.cu
struct RecordDelete { void operator()(SamsState *) const; void operator()(MolTables *) const; };
template <typename T> using RecordPtr = std::unique_ptr<T, RecordDelete>;

// ---- MT19937 stream resident on the device (numba's / numpy's generator restated) ---------------------
struct MTStream {
    DevBuf<uint32_t> d_window;   // last 624 raw words x_n .. x_{n+623}
    DevBuf<uint32_t> d_words;    // tempered outputs not yet consumed: d_words[0..avail)
    DevBuf<uint32_t> d_words_alt;
    size_t cap = 0;
    size_t avail = 0;
    uint64_t consumed = 0;  // words consumed since seeding
    bool seeded = false;
};

struct SlotRec {        // one 2-word "slot" of the stream, state independent (pow2 K fast path)
    uint32_t ij;        // i | j << 16 (masked replica indices)
    uint32_t backmask;  // bit 31-b: slot s-1-b shares a replica index with slot s (b = 0..30)
    double logU;        // log of the uniform the two words of THIS slot would produce
};

struct MixCtl {          // device-resident control block of the resumable mixing kernels
    long long head;      // in: first unconsumed word (K not a power of two) / slot (power-of-two K);  out: same after the call
    long long remaining; // attempts still to do
    int status;          // 0 done, 1 need more words
    int rounds;          // statistics: speculation rounds executed
    long long slow_exp;  // statistics: exact exp() fallbacks
    long long log_count; // entries written to the commit log by this launch
    long long aux;       // k_mix_walk2 / k_mix_walk2c: record reached (extent of their sparse commit log)
};

// How a swap-all pass walks the chain (mix_plan in rx_mix.cu): coordinates and filter choose the records and the walkers.
enum MixCoords { MIX_LOOP, MIX_SLOTS, MIX_CANDS };   // the plain loop alone, slots (power-of-two K), candidate indices
struct MixPlan {
    MixCoords coords;
    bool filter;      // a filter walker takes the bulk of the pass, on SlotRec2 records (else SlotRec / CandRec)
    int head_unit;    // stream words per unit of MixCtl::head
    int smem_tail;    // dynamic shared memory of the kernel that finishes the pass (the bulk walkers take WALK_SMEM)
    bool operator==(const MixPlan &o) const {
        return coords == o.coords && filter == o.filter && head_unit == o.head_unit && smem_tail == o.smem_tail;
    }
};

struct rx_state_move {
    double dt = 0, gamma = 0;
    int n_steps = 0, reassign = 0;
    char program[RX_MAX_PROGRAM] = {0};
    bool set = false;
    bool hmc = false;   // hybrid Monte Carlo (program "VRV", gamma 0): rx_set_state_hmc_integrator
};

struct rx_engine {
    rx_config cfg;
    int k0 = 0, kloc = 0;  // owned replicas [k0, k0+kloc)
    int n_sm = 0;          // multiprocessors of cfg.device
    int smem_optin = 0;    // opt-in shared memory per block of cfg.device (bytes)
    cudaStream_t stream = nullptr, stream_rng = nullptr;
    cudaEvent_t ev[8] = {};
    cudaEvent_t ev_user[2] = {};
    long long mix_stats[6] = {0, 0, 0, 0, 0, 0};   // rounds, exact-exp, passes, words, walker us, prepare-wait us
    cudaEvent_t ev_walk[2] = {};
    // particles
    DevBuf<float4> d_atom;        // (sigma, sqrt_eps, inv_mass, alch ? 1 : 0), or the region id (0, 1, 2) with two regions
    DevBuf<double4> d_atom_d;     // (sigma, eps, mass, alch or region id)
    std::vector<float4> h_atom;   // host copies of both (rx_set_alchemical_regions rewrites their w)
    std::vector<double4> h_atom_d;
    int n_alch = 0;
    DevBuf<int> d_alch_list;      // indices of the alchemical atoms (of either region)
    // two alchemical regions (rx_set_alchemical_regions): the two-region kernel instantiations run, and their pair rules
    // read the annihilate flags as bit 0 (region 1) and bit 1 (region 2) of DynParams / EnParams::annihilate
    bool two_regions = false;
    int annihilate_mask = 0;
    bool have_particles = false, have_states = false, have_integrator = false;
    DevBuf<StateDev> d_states;
    std::vector<StateDev> h_states;
    // replica state
    DevBuf<float4> d_pos, d_vel;                // [kloc][N]
    DevBuf<float4> d_pos_snap, d_vel_snap;      // start-of-iteration copy for the NaN restart policy
    DevBuf<int> d_retry;                        // [K] replicas to propagate again
    bool have_snapshot = false;
    DevBuf<double> d_io;                        // staging for set/get: [kloc][N][3]
    PinnedBuf<double> h_io;                     // pinned host staging of the same size
    std::vector<std::pair<const char *, size_t>> pinned;   // caller buffers registered with rx_pin_host_memory
    DevBuf<int> d_perm;                         // [K] replica -> state
    DevBuf<double> d_u;                         // [K][M]
    DevBuf<unsigned long long> d_nacc, d_nprop;  // [M][M]
    DevBuf<double> d_pot, d_kin;                // [K]
    DevBuf<int> d_nan;                          // [K]
    DevBuf<int> d_err;                          // device error flag (capacity overflow, ...)
    // energy kernel scratch: lambda-controlled pairs per owned replica
    DevBuf<double2> d_pairs;   // [kloc][pair_cap]: ((r / sigma)^c, negative in region 2; 4 eps S(r)) of k_energy_rows
    int pair_cap = 0;
    // integrator
    double dt = 0, gamma = 0;
    int n_steps = 0;
    char program[RX_MAX_PROGRAM] = {0};
    bool hmc = false;                        // the engine's move is hybrid Monte Carlo (rx_set_hmc_integrator)
    DevBuf<ulonglong2> d_hmc_stats;          // [kloc] (accepted, trials) of HMC, cumulative
    DevBuf<double2> d_hmc_energy;            // [kloc] (Eold, Enew) of each owned replica's last HMC trial
    RecordPtr<MolTables> mol;                // the molecule of a RX_SYSTEM_MOLECULE engine: device tables, MolDev and MolGB
    std::vector<rx_state_move> state_moves;   // per-state moves (empty: one move for all states)
    bool state_moves_dirty = false;
    DevBuf<MoveDev> d_moves;
    std::vector<int> mol_cluster;            // constraint cluster of each atom of a molecule (-1: unconstrained)
    // Monte Carlo moves (rx_set_state_mc_moves): [M][RX_MAX_MC_MOVES] records, kind -1 where a state has fewer moves
    std::vector<int32_t> mc_atoms;           // rx_set_mc_subsets
    DevBuf<int32_t> d_mc_atoms;
    std::vector<rx_mc_move> mc_moves;
    DevBuf<rx_mc_move> d_mc_moves;
    int mc_slots = 0;                        // the most moves any state has: launches per propagation
    DevBuf<unsigned long long> d_mc_acc, d_mc_prop;   // [M][RX_MAX_MC_MOVES]
    DevBuf<double> d_mc_du;                  // [kloc][RX_MAX_MC_MOVES]: dU of each owned replica's last proposal per slot
    // mixing
    MTStream streams[2];
    DevBuf<uint4> d_slots;      // the 16-byte records of a pass: SlotRec, SlotRec2 or CandRec
    size_t slots_cap = 0;
    DevBuf<MixCtl> d_ctl;
    DevBuf<uint32_t> d_log;      // commit log of the walker: packed (si, sj, accepted)
    DevBuf<uint32_t> d_slotlog;      // sparse commit log of k_mix_walk2: one word per slot
    DevBuf<uint32_t> d_cpos;         // k_mix_walk2c / k_mix_walk_cand: word position of every candidate of the pass
    DevBuf<uint32_t> d_ctile;        // ... candidates per tile / their exclusive scan, then [last] = number of candidates
    size_t ctile_cap = 0;
    DevBuf<unsigned char> d_filt;      // 24-bit row image of u for the K=256 walker
    DevBuf<double> d_filt_scale;       // [K] scales + [K] row abs-max
    struct {
        bool valid = false;       // words + records for the next swap-all call were produced on stream_rng ...
        MixPlan plan = {};        // ... for this plan
        size_t avail = 0;         // ... over this many stream words
    } prepared;
    size_t last_consumed = 0;     // words the previous swap-all call consumed (sizes the generate-ahead)
    cudaEvent_t ev_prepared = nullptr, ev_consumed = nullptr;
    RecordPtr<SamsState> sams;    // SamsState (rx_sams.cuh): device-resident logZ / weights / histogram of a SAMSSampler
    // timing
    double phase_ms[4] = {0, 0, 0, 0};
    long long phase_launches[4] = {0, 0, 0, 0};
    // constant pressure (rx_set_pressures): per owned replica box (x, y, z, -) and barostat state, per state (p, c)
    bool npt = false;
    DevBuf<double4> d_box, d_box_snap;
    DevBuf<rx_barostat_state> d_baro, d_baro_snap;
    DevBuf<double2> d_npt;
    // anisotropic barostat (rx_set_anisotropic_barostat): per owned replica per-axis state; the step counter stays in d_baro
    bool aniso = false;
    DevBuf<rx_anisotropic_barostat_state> d_aniso, d_aniso_snap;
    // energies of the last rx_compute_energies_at* call, [K][u_at_cols] after the all-gather
    DevBuf<double> d_u_at;
    size_t u_at_cap = 0;
    int u_at_cols = 0;
    // energy history (rx_history_*): row t is iteration t, [K][M + hist_u] (the sampled states, then the unsampled ones)
    DevBuf<double> d_hist;
    size_t hist_cap = 0;          // doubles
    long long hist_len = 0;       // rows
    int hist_u = 0;
    // nccl
    void *nccl_lib = nullptr;
    void *nccl_comm = nullptr;
    std::string err;
};

extern thread_local std::string g_rx_create_error;

#define RX_CHECK_CUDA(h, call)                                                                     \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            (h)->err = std::string(#call) + ": " + cudaGetErrorString(_e);                         \
            return RX_ERR_CUDA;                                                                    \
        }                                                                                          \
    } while (0)

#define RX_FAIL(h, code, msg)     \
    do {                          \
        (h)->err = (msg);         \
        return (code);            \
    } while (0)

// phase timing helper: records events around a phase on h->stream
struct PhaseTimer {
    rx_engine *h;
    int phase;
    PhaseTimer(rx_engine *h_, int p) : h(h_), phase(p) { cudaEventRecord(h->ev[2 * p], h->stream); }
    void stop(int launches) {
        cudaEventRecord(h->ev[2 * phase + 1], h->stream);
        h->phase_launches[phase] += launches;
    }
    void accumulate() {  // call after a stream sync
        float ms = 0;
        if (cudaEventElapsedTime(&ms, h->ev[2 * phase], h->ev[2 * phase + 1]) == cudaSuccess) h->phase_ms[phase] += ms;
    }
};

// ---- implemented in rx_mix.cu ----
int rxi_mix_seed(rx_engine *h, int stream, uint32_t seed);
int rxi_mix_skip(rx_engine *h, int stream, unsigned long long n);
int rxi_selftest_exp(rx_engine *h, const double *x, double *y, int n);
int rxi_mix_swap_all(rx_engine *h, long long nswap, int *launches);
int rxi_mix_swap_neighbors(rx_engine *h, int *launches);
int rxi_sams_set(rx_engine *h, const rx_sams_config *c, const double *log_target, const double *logZ, const int64_t *histogram);
int rxi_sams_step(rx_engine *h, long long iteration, int update, int *launches);
int rxi_sams_get(rx_engine *h, double *logZ, double *log_weights, int64_t *histogram, int32_t *stage, int64_t *t0, double *gamma,
                 int64_t *states, int64_t *previous_states);
int rxi_sams_set_histogram(rx_engine *h, const int64_t *histogram);

// ---- implemented in rx_dynamics.cu ----
int rxi_propagate(rx_engine *h, uint64_t seed, uint64_t iteration, int reassign, int *launches, const int *d_only = nullptr);
int rxi_plan_propagate(const rx_propagate_query *q, rx_propagate_plan *out, std::string &err);   // host arithmetic only
int rxi_upload_state_moves(rx_engine *h);
int rxi_set_molecule(rx_engine *h, const rx_molecule *mol);
int rxi_set_implicit_solvent(rx_engine *h, const rx_gbsa *s);
int rxi_mc_moves(rx_engine *h, uint64_t seed, uint64_t iteration, int *launches);   // one launch per MC slot (rx_mc.cuh)
int rxi_snapshot_state(rx_engine *h);   // positions + velocities at the start of a propagation
int rxi_restore_failed(rx_engine *h);   // replicas with a NaN flag go back to the snapshot; d_retry = the flags
int rxi_compute_energy_rows(rx_engine *h, int *launches);  // fills d_u rows [k0, k0+kloc)
int rxi_compute_energy_rows_at(rx_engine *h, const StateDev *d_states, int n_states, double *d_out, int *launches,
                               const double2 *d_npt_tab = nullptr);   // NPT: (pressure, dispersion) of those states
int rxi_randomize_velocities(rx_engine *h, uint64_t seed, uint64_t stream_id);
int rxi_minimize(rx_engine *h, double tolerance, int max_iterations, double *d_rms, int *d_iters);  // [K] each
int rxi_convert_in(rx_engine *h, float4 *dst, int first_local, int count, const double *host_xyz, bool is_vel);
int rxi_convert_out(rx_engine *h, const float4 *src, int first_local, int count, double *host_xyz, bool wrap);

// ---- implemented in rx_api.cu ----
bool rxi_is_pinned(const rx_engine *h, const void *p, size_t bytes);
int rxi_allgather_energies(rx_engine *h);
int rxi_allgather_rows(rx_engine *h, double *d_matrix, int n_cols);
