/*
 * rx_b200.h -- C ABI of librx_b200.so, the H100-native replica-exchange engine.
 *
 * This is the drop-in boundary for the hot path of choderalab/openmmtools'
 * multistate.ReplicaExchangeSampler (mix -> propagate -> energies; reference:
 * openmmtools/multistate/multistatesampler.py:766-804).  The reference has no native/FFI boundary for this
 * path (it is Python over OpenMM); its extension points are the three sampler hooks and the MCMCMove.apply
 * interface (SURVEY.md section 8b).  Each entry point below names the reference code it replaces; the
 * Python-side binding a maintainer would add is shown in INTEGRATION.md and shipped in
 * openmmtools_b200/_engine.py.
 *
 * Conventions: C linkage, POD structs, caller-owned host buffers (C-contiguous), md units
 * (nm, ps, amu, kJ/mol, K).  Every call returns 0 on success or a negative rx_status; the message is
 * available from rx_last_error().  No exceptions cross the ABI.  One engine = one GPU = one host thread;
 * calls are not re-entrant.  Every call synchronises with the device before returning unless noted.
 */
#ifndef RX_B200_H
#define RX_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RX_ABI_VERSION 1
#if defined(__GNUC__)
#define RX_API __attribute__((visibility("default")))
#else
#define RX_API
#endif

typedef struct rx_engine rx_engine;

enum rx_status {
    RX_OK = 0,
    RX_ERR_INVALID = -1,     /* bad argument / call order          -> ValueError / RuntimeError        */
    RX_ERR_CUDA = -2,        /* CUDA runtime failure               -> RuntimeError                     */
    RX_ERR_NAN = -3,         /* NaN positions/energies             -> SimulationNaNError / IntegratorMoveError */
    RX_ERR_UNSUPPORTED = -4, /* feature outside the hot path       -> NotImplementedError              */
    RX_ERR_COMM = -5,        /* NCCL failure                       -> RuntimeError                     */
    RX_ERR_CAPACITY = -6     /* an internal list overflowed        -> RuntimeError                     */
};

enum rx_system_kind {
    RX_SYSTEM_NONE = 0,     /* mixing only: energies are supplied with rx_set_energies                */
    RX_SYSTEM_LJ_ALCH = 1,  /* testsystems.LennardJonesFluid (testsystems.py:1872-2030) through
                               alchemy.AbsoluteAlchemicalFactory (alchemy.py:1539-2038): switched LJ +
                               soft-core sterics, per-atom sigma/epsilon/mass, rectangular periodic
                               box (box[0..2] = x, y, z edges)                                         */
    RX_SYSTEM_HARMONIC = 2, /* testsystems.HarmonicOscillator (testsystems.py:761-788), per-state K/x0/U0 */
    RX_SYSTEM_MOLECULE = 3  /* a small molecule in vacuum (<= 32 atoms), e.g. testsystems.AlanineDipeptideVacuum
                               (testsystems.py:3352-3388): harmonic bonds and angles, periodic torsions, all-pairs
                               Coulomb + Lennard-Jones with exclusions and scaled 1-4 pairs, distance constraints;
                               states differ in temperature only (ParallelTemperingSampler)                  */
};

typedef struct {
    int32_t abi_version;      /* RX_ABI_VERSION */
    int32_t system_kind;      /* rx_system_kind */
    int32_t n_replicas;       /* K, global */
    int32_t n_states;         /* M (== K for ReplicaExchangeSampler) */
    int32_t n_atoms;          /* N */
    int32_t device;           /* CUDA ordinal */
    int32_t rank;             /* replica shard owner: this engine owns replicas [rank*K/world, (rank+1)*K/world) */
    int32_t world_size;       /* 1 = single GPU */
    double box[3];            /* cubic/rectangular periodic box edge lengths (LJ) */
    double r_cutoff;          /* NonbondedForce cutoff (testsystems.py:1981)          */
    double r_switch;          /* switching distance (testsystems.py:1989)             */
    int32_t use_switch;       /* 1: OpenMM switching function on [r_switch, r_cutoff] */
    int32_t annihilate_sterics; /* AlchemicalRegion.annihilate_sterics (alchemy.py:423) */
    double softcore_alpha, softcore_a, softcore_b, softcore_c; /* alchemy.py:424 */
} rx_config;

/* One thermodynamic state (states.ThermodynamicState + alchemy.AlchemicalState / HO parameters). */
typedef struct {
    double temperature;      /* K; beta = 1/(kB*T), kB = 8.31446261815324e-3 kJ/mol/K (constants.py:7)  */
    double lambda_sterics;   /* AlchemicalState.lambda_sterics (alchemy.py:207-225)                       */
    double energy_offset;    /* kJ/mol added to U in this state (dispersion corrections, U0)              */
    double ho_K;             /* kJ/mol/nm^2 */
    double ho_x0[3];         /* nm */
} rx_state_params;

/* ---- lifecycle ------------------------------------------------------------------------------------ */
/* Replaces: MultiStateSampler.create/_pre_write_create (multistatesampler.py:537-609,836-926) +
 * ContextCache.get_context (cache.py:378-461): allocates the resident device state once.               */
RX_API int rx_create(const rx_config *cfg, rx_engine **out);
RX_API void rx_destroy(rx_engine *h);
/* h may be NULL to read the error of a failed rx_create. Pointer valid until the next call. */
RX_API const char *rx_last_error(const rx_engine *h);
RX_API int rx_abi_version(void);

/* The force field of a RX_SYSTEM_MOLECULE engine, in md units (nm, kJ/mol, amu, e, rad), as
 * openmm.app.AmberPrmtopFile.createSystem(implicitSolvent=None, nonbondedCutoff=None, constraints=...) defines it for
 * testsystems.AlanineDipeptideVacuum (openmmtools/testsystems.py:3375-3388).  Arrays are caller-owned and copied.
 *   bonds[n][4]       i, j, K, r0            1/2 K (r - r0)^2        (constrained bonds are NOT listed here)
 *   angles[n][5]      i, j, k, K, theta0     1/2 K (theta - theta0)^2
 *   torsions[n][7]    i, j, k, l, n, phase, k    k (1 + cos(n phi - phase))
 *   exclusions[n][2]  pairs without nonbonded interaction (1-2, 1-3)
 *   exceptions[n][5]  i, j, q_i q_j, sigma, epsilon   replacing the pair's interaction (scaled 1-4 pairs)
 *   constraints[n][3] i, j, distance
 * All other pairs interact by 138.935456 q_i q_j / r + 4 eps_ij ((s_ij/r)^12 - (s_ij/r)^6), Lorentz-Berthelot s_ij, eps_ij.
 * remove_cm_motion: the centre-of-mass velocity is removed at the start of every integration step (CMMotionRemover).
 * constraint_tolerance: relative tolerance of the constraint solvers (integrators.py: constraint_tolerance, 1e-8). */
typedef struct {
    int32_t n_bonds, n_angles, n_torsions, n_exclusions, n_exceptions, n_constraints, remove_cm_motion, reserved;
    double constraint_tolerance;
    const double *mass, *charge, *sigma, *epsilon;   /* [n_atoms] */
    const double *bonds, *angles, *torsions;
    const int64_t *exclusions;
    const double *exceptions, *constraints;
} rx_molecule;

/* ---- static tables -------------------------------------------------------------------------------- */
/* per-atom sigma (nm), epsilon (kJ/mol), mass (amu), alchemical mask; for RX_SYSTEM_HARMONIC only mass. */
RX_API int rx_set_particles(rx_engine *h, const double *sigma, const double *epsilon, const double *mass,
                     const uint8_t *alchemical_mask);
RX_API int rx_set_states(rx_engine *h, const rx_state_params *states /* [n_states] */);
/* Two alchemical regions (RX_SYSTEM_LJ_ALCH).  Replaces AbsoluteAlchemicalFactory.create_alchemical_system with a list
 * of two AlchemicalRegions and no alchemical_regions_interactions (alchemy.py:637-754, 1539-2038): region[i] is 0 for the
 * environment, 1 or 2 for the atoms of the first or second region (their epsilons are zeroed in the NonbondedForce,
 * :1903-1909); environment x region r pairs are soft-core sterics driven by region r's lambda_sterics<suffix>
 * (:1774-1775, 1915), r x r pairs the same expression with lambda 1 unless annihilate_r (:1776-1777, 1919), and pairs
 * across the two regions have no interaction (no force covers them, :1684-1685).  Both regions use the soft-core
 * constants of rx_config (OpenMM keeps one value per global parameter name, :2009-2017); annihilate_1/annihilate_2
 * replace rx_config.annihilate_sterics.  Call after rx_set_particles (which returns the engine to one region); the
 * engine then runs the two-region kernel instantiations.
 * rx_set_states_region2  lambda_sterics of the second region [n_states] (GlobalParameterState with a
 *                        parameters_name_suffix, states.py:3276-3280, 3830-3898); rx_set_states resets it to 1, so call
 *                        it after every rx_set_states.  rx_state_params.lambda_sterics is the first region's lambda. */
RX_API int rx_set_alchemical_regions(rx_engine *h, const uint8_t *region /*[N]*/, int32_t annihilate_1, int32_t annihilate_2);
RX_API int rx_set_states_region2(rx_engine *h, const double *lambda_sterics_2 /*[n_states]*/);
/* RX_SYSTEM_MOLECULE: the particles and the force field at once (instead of rx_set_particles).
 * Replaces: the System built by AmberPrmtopFile.createSystem for AlanineDipeptideVacuum, testsystems.py:3375-3388.
 * RX_ERR_UNSUPPORTED (and no molecule set) when the term tables need more shared memory than a block of the device can
 * have (each torsion term takes 236 bytes of the 227 KB of an H100 block: decane with three terms per torsion needs 95 KB); a refused call leaves the engine without a molecule. */
RX_API int rx_set_molecule(rx_engine *h, const rx_molecule *molecule);
/* OBC generalized Born implicit solvent for the molecule of the last rx_set_molecule (which returns the engine to vacuum):
 * what AmberPrmtopFile.createSystem(implicitSolvent=OBC1|OBC2, nonbondedCutoff=None) adds, without salt.  For atom i
 * (rt = radius - offset, sr = scale rt):
 *   I_i = sum_{j != i} 1/2 [1/L - 1/U + 1/4 (r - sr_j^2/r)(1/U^2 - 1/L^2) + 1/2 ln(L/U)/r]   over pairs with r + sr_j > rt_i
 *         (U = r + sr_j, L = max(rt_i, |r - sr_j|); every pair, excluded and 1-4 pairs included; no engulfment term),
 *   B_i = 1 / (1/rt_i - tanh(alpha psi - beta psi^2 + gamma psi^3) / radius_i),  psi = I_i rt_i,
 *   E   = sum_i [1/2 P q_i^2 / B_i + 4 pi sa_energy (radius_i + probe_radius)^2 (radius_i / B_i)^6]
 *       + sum_{i<j} P q_i q_j / sqrt(r^2 + B_i B_j exp(-r^2 / (4 B_i B_j))),   P = -138.935456 (1/solute - 1/solvent dielectric).
 * OBC1: alpha, beta, gamma = 0.8, 0, 2.909125; OBC2: 1.0, 0.8, 4.85; offset 0.009 nm; sa_energy 2.25936 kJ/mol/nm^2 (0: no
 * non-polar term), probe_radius 0.14 nm.  RX_ERR_INVALID for a radius <= 0 or <= offset, a negative scale, or an engine
 * without a molecule; RX_ERR_UNSUPPORTED when the tables no longer fit in a block (the propagation kernel adds
 * 8 (4 n^2 + 3 n) bytes to the molecule's, 33 KB at 32 atoms); a refused call leaves the engine as it was. */
typedef struct {
    const double *radius, *scale;   /* [n_atoms]: nm, dimensionless */
    double alpha, beta, gamma, offset;
    double solute_dielectric, solvent_dielectric;
    double sa_energy, probe_radius;   /* kJ/mol/nm^2, nm */
} rx_gbsa;
RX_API int rx_set_implicit_solvent(rx_engine *h, const rx_gbsa *gbsa);
/* LangevinSplittingDynamicsMove parameters (mcmc.py:1280-1291) / LangevinIntegrator (integrators.py:1071-1158):
 * timestep (ps), collision_rate (1/ps), n_steps, splitting with the spaces removed, e.g. "VRORV".        */
RX_API int rx_set_integrator(rx_engine *h, double timestep, double collision_rate, int32_t n_steps,
                      const char *splitting);

/* One move per thermodynamic state: a replica is propagated with the move of the state it is in.
 * Replaces: the per-state mcmc_moves list of MultiStateSampler, openmmtools/multistate/multistatesampler.py:906-910 (one deep
 * copy per state) and its use in _propagate_replica, :1311-1322 (mcmc_move = self._mcmc_moves[thermodynamic_state_id]).
 * Call after rx_set_integrator (the move of every state not set here), once per state whose move differs;
 * reassign_velocities is that move's flag (the `reassign_velocities` argument of rx_propagate is then ignored).
 * rx_set_integrator again returns to one move for all states. */
RX_API int rx_set_state_integrator(rx_engine *h, int32_t state, double timestep, double collision_rate, int32_t n_steps,
                                   const char *splitting, int32_t reassign_velocities);

/* ---- Monte Carlo rigid-body moves (MCDisplacementMove, MCRotationMove: mcmc.py:810-970, 1704-1911) ------------------ */
/* Up to RX_MAX_MC_MOVES Metropolized moves per thermodynamic state, applied in order to every replica in that state at the
 * start of rx_propagate (before its snapshot, so rx_propagate_retry reruns the dynamics only, from the post-MC state) and of
 * every iteration of rx_run_iterations / rx_sams_run_iterations.  One proposal per move and replica:
 *   RX_MC_DISPLACEMENT  the subset moves by sigma_nm * (three standard normals);
 *   RX_MC_ROTATION      the subset turns about its geometric centre by a uniform random rotation (Shoemake's quaternion).
 *                       On a periodic box the subset is first made whole by minimum image relative to its first atom, and
 *                       the proposal is rejected when a rotated offset from that atom reaches half a box edge.
 * The proposal is accepted iff dU is finite and beta dU <= 0 or u < exp(-beta dU), beta and U of the replica's state; positions
 * stay f32 (a molecule's f64), and a periodic system's are wrapped into the box as rx_propagate wraps them.  Randoms: Philox4x32-10 keyed as rx_propagate's noise, counter (slot, 0xE0000000, replica,
 * iteration) for the proposal and (slot, 0xE0000001, replica, iteration) for u.
 * rx_set_mc_subsets      the atom indices every move's subset points into (subset_offset, subset_len); replaces the previous
 *                        array and removes every move set so far.
 * rx_set_state_mc_moves  the n moves of `state` (-1: every state); n = 0 removes them.  RX_ERR_UNSUPPORTED when a subset of a
 *                        molecule contains part of a constraint cluster (a rigid move keeps the constraints only when it moves
 *                        whole clusters).
 * rx_get_mc_statistics / rx_set_mc_statistics  accepted and proposed counts [M][RX_MAX_MC_MOVES] of the replicas this engine
 *                        owns (with world_size > 1, the totals are the sums over the ranks). */
#define RX_MAX_MC_MOVES 4
enum rx_mc_kind { RX_MC_DISPLACEMENT = 0, RX_MC_ROTATION = 1 };
typedef struct {
    int32_t kind;              /* rx_mc_kind */
    int32_t subset_offset, subset_len;
    int32_t reserved;
    double sigma_nm;           /* RX_MC_DISPLACEMENT: standard deviation of each component of the displacement */
} rx_mc_move;
RX_API int rx_set_mc_subsets(rx_engine *h, const int32_t *atoms, int32_t n);
RX_API int rx_set_state_mc_moves(rx_engine *h, int32_t state, int32_t n, const rx_mc_move *moves);
RX_API int rx_get_mc_statistics(rx_engine *h, int64_t *accepted, int64_t *proposed);
RX_API int rx_set_mc_statistics(rx_engine *h, const int64_t *accepted, const int64_t *proposed);
/* Diagnostic: du[K][RX_MAX_MC_MOVES] (kJ/mol) of the last proposal of every owned replica in every move slot -- the energy
 * change the acceptance test used, the difference of the replica's own rows of rx_compute_energies at the proposed and the
 * current positions, divided by beta; NaN where no energy was computed (a rejected rotation on a periodic box, an unused
 * slot, a replica this engine does not own). */
RX_API int rx_get_mc_energy_changes(rx_engine *h, double *du);

/* ---- replica state I/O (SamplerState.apply_to_context / update_from_context, states.py:2215-2279) -- */
/* xyz: [count][N][3] doubles, global replica indices; replicas not owned by this engine are skipped.    */
RX_API int rx_set_positions(rx_engine *h, int32_t first, int32_t count, const double *xyz);
RX_API int rx_set_velocities(rx_engine *h, int32_t first, int32_t count, const double *xyz);
RX_API int rx_get_positions(rx_engine *h, int32_t first, int32_t count, double *xyz);
RX_API int rx_get_velocities(rx_engine *h, int32_t first, int32_t count, double *xyz);
/* potential (kJ/mol, in the replica's current state) and kinetic energy after the last propagate.       */
/* Page-lock a caller buffer so that rx_set_* / rx_get_* on (parts of) it copy directly, without the engine's staging
 * buffer (the host-resident SamplerState arrays of MultiStateSampler, multistatesampler.py:1296-1337 keeps them on the
 * host between iterations).  Unregistered by rx_unpin_host_memory or rx_destroy.                                  */
RX_API int rx_pin_host_memory(rx_engine *h, void *buffer, uint64_t bytes);
RX_API int rx_unpin_host_memory(rx_engine *h, void *buffer);

RX_API int rx_get_replica_energies(rx_engine *h, double *potential /*[K] or NULL*/, double *kinetic /*[K] or NULL*/);
/* context.setVelocitiesToTemperature (mcmc.py:711): v = sqrt(kB T/m) N(0,1) for every owned replica.     */
RX_API int rx_randomize_velocities(rx_engine *h, uint64_t seed, uint64_t stream);
/* Replaces MultiStateSampler.minimize (multistatesampler.py:612-647) -> _minimize_replica (:1339-1402): FIRE descent
 * of every owned replica in its current state until the RMS force component is below `tolerance` (kJ/mol/nm) or
 * `max_iterations` steps were taken (0: the built-in cap of 20000).  Velocities are not touched.  rms_force[K] and
 * iterations[K] (either may be NULL) are filled for the replicas this rank owns, zero elsewhere.                  */
RX_API int rx_minimize(rx_engine *h, double tolerance, int32_t max_iterations, double *rms_force, int32_t *iterations);

/* replica -> state map (MultiStateSampler._replica_thermodynamic_states, multistatesampler.py:895)       */
RX_API int rx_set_replica_states(rx_engine *h, const int64_t *states /*[K]*/);
RX_API int rx_get_replica_states(rx_engine *h, int64_t *states /*[K]*/);

/* ---- the three phases ----------------------------------------------------------------------------- */
/* Replaces MultiStateSampler._propagate_replicas (multistatesampler.py:1287-1337) ->
 * BaseIntegratorMove.apply (mcmc.py:668-776) -> integrator.step(n_steps) (mcmc.py:719).
 * Noise is Philox4x32-10 keyed by (seed; iteration, global replica, atom, step), so trajectories do not
 * depend on the number of GPUs.  nan_flags[K] (may be NULL) gets 1 for replicas whose state went NaN.
 * Replicas of up to 4096 atoms (RX_SYSTEM_LJ_ALCH; above 1024 a replica spans a cluster of 2, 4 or 8 thread blocks) or
 * 1024 atoms (RX_SYSTEM_HARMONIC); larger ones return RX_ERR_UNSUPPORTED here and in rx_minimize.        */
RX_API int rx_propagate(rx_engine *h, uint64_t seed, uint64_t iteration, int32_t reassign_velocities,
                 int32_t *nan_flags);
/* Replaces the restart loop of BaseIntegratorMove.apply (mcmc.py:706-759, n_restart_attempts): after rx_propagate
 * returned RX_ERR_NAN, the replicas whose flag is set go back to the state they had when that call began (a
 * device-side snapshot) and are propagated again -- pass another seed for other noise; replicas that came through
 * are not touched.                                                                                         */
RX_API int rx_propagate_retry(rx_engine *h, uint64_t seed, uint64_t iteration, int32_t reassign_velocities,
                 int32_t *nan_flags);

/* Replaces MultiStateSampler._compute_energies (multistatesampler.py:1436-1494) ->
 * ThermodynamicState.reduced_potential_at_states (states.py:911-992).  Fills the device-resident
 * u[K][M]; with world_size > 1 the rows are all-gathered over NCCL.  u_out (may be NULL): [K][M].        */
RX_API int rx_compute_energies(rx_engine *h, double *u_out);
/* Reduced potentials of every replica at `n` OTHER states (MultiStateSampler's unsampled_thermodynamic_states,
 * multistatesampler.py:1452-1456,1489-1494; ThermodynamicState.reduced_potential_at_states, states.py:911-992): same
 * kernel, temporary state table, does not touch the resident matrix.  u_out: [K][n].                                */
RX_API int rx_compute_energies_at(rx_engine *h, const rx_state_params *states, int32_t n, double *u_out);
RX_API int rx_set_energies(rx_engine *h, const double *u /*[K][M]*/);
RX_API int rx_get_energies(rx_engine *h, double *u /*[K][M]*/);

/* Replaces ReplicaExchangeSampler._mix_replicas (replicaexchange.py:255-292).
 * swap-all: bit-exact restatement of _mix_all_replicas_numba (replicaexchange.py:294-349) on the numba
 * MT19937 stream `RX_STREAM_NUMBA`; swap-neighbors: _mix_neighboring_replicas (:366-380) on the numpy
 * RandomState stream `RX_STREAM_NUMPY`.  Count matrices are zeroed by the call (as :261-262 does) and
 * returned if the pointers are non-NULL ([M][M] int64).                                                   */
enum rx_rng_stream { RX_STREAM_NUMBA = 0, RX_STREAM_NUMPY = 1 };
RX_API int rx_mix_seed(rx_engine *h, int32_t stream, uint32_t seed);         /* np.random.seed(seed) semantics */
RX_API int rx_mix_swap_all(rx_engine *h, int64_t nswap_attempts, int64_t *states_out /*[K] or NULL*/,
                    int64_t *n_accepted /*[M][M] or NULL*/, int64_t *n_proposed /*[M][M] or NULL*/);
RX_API int rx_mix_swap_neighbors(rx_engine *h, int64_t *states_out, int64_t *n_accepted, int64_t *n_proposed);
RX_API int rx_get_mix_counts(rx_engine *h, int64_t *n_accepted, int64_t *n_proposed);
/* MT words consumed so far on a stream (for checkpoints: state = seed + position); rx_mix_skip advances a freshly
 * seeded stream by n words (resume: rx_mix_seed(seed) + rx_mix_skip(position)).                              */
RX_API int rx_mix_skip(rx_engine *h, int32_t stream, uint64_t n_words);
RX_API int rx_mix_stream_position(rx_engine *h, int32_t stream, uint64_t *words_consumed);

/* Fused hot loop: n_iterations x (mix -> propagate -> energies), multistatesampler.py:776-782, with no host
 * round trip in between.  mixing: 0 none, 1 swap-all (nswap = K^3), 2 swap-neighbors.                     */
RX_API int rx_run_iterations(rx_engine *h, int32_t n_iterations, int32_t mixing, uint64_t seed,
                      uint64_t first_iteration, int32_t reassign_velocities);

/* Replaces SAMSSampler._mix_replicas (/root/reference/openmmtools/multistate/sams.py:395-437): the global state jump
 * (_global_jump, :477-501), the stage schedule (_update_stage, :564-604), the online logZ update (_update_logZ_estimates,
 * :606-681) and log_weights = log_target - logZ (:683-691) in ONE kernel on the resident K x M energy matrix; logZ, weights,
 * state histogram, stage and t0 stay on the device between iterations.  The jump draws numpy RandomState.choice's uniform (one
 * random_sample per replica) from the RX_STREAM_NUMPY stream (rx_mix_seed).
 *   rx_sams_set   configuration + initial logZ [M], log target probabilities [M], state histogram [M] (NULL: zeros)
 *   rx_sams_step  one jump for every replica (+ the weight update when update_weights != 0; sams.py:429-435 skips it during
 *                 equilibration); histogram: the host's state histogram to use (NULL: the device's own count, which the kernel
 *                 advances by the new states of every call); results through rx_sams_get
 *   rx_sams_run_iterations  n x (jump + update -> propagate -> energies), no host round trip                             */
typedef struct rx_sams_config {
    double gamma0, flatness_threshold;
    int32_t weight_update_method;   /* 0 'optimal', 1 'rao-blackwellized' */
    int32_t two_stage;              /* update_stages == 'two-stage' */
    int32_t flatness_criteria;      /* 0 'minimum-visits', 1 'histogram-flatness', 2 'logZ-flatness' */
    int32_t stage;                  /* current stage (0 | 1) and t0, sams.py:318-328 */
    int64_t t0;
} rx_sams_config;
RX_API int rx_sams_set(rx_engine *h, const rx_sams_config *config, const double *log_target_probabilities, const double *logZ,
                       const int64_t *histogram);
RX_API int rx_sams_step(rx_engine *h, int64_t iteration, int32_t update_weights, const int64_t *histogram);
RX_API int rx_sams_get(rx_engine *h, double *logZ, double *log_weights, int64_t *histogram, int32_t *stage, int64_t *t0,
                       double *gamma, int64_t *states /*[K]*/, int64_t *previous_states /*[K]*/);
RX_API int rx_sams_run_iterations(rx_engine *h, int32_t n_iterations, uint64_t seed, uint64_t first_iteration,
                                  int32_t reassign_velocities);

/* Device-side phase timings (CUDA events) of the last rx_run_iterations / phase calls, in ms:
 * [0] mix, [1] propagate, [2] energies (incl. allgather), [3] rng-stream generation, accumulated;
 * counts[i] = number of launches of my kernels in phase i.                                                */
RX_API int rx_get_phase_times(rx_engine *h, double ms[4], int64_t counts[4], int32_t reset);

/* CUDA-event stopwatch on the engine's stream: rx_timer_mark(h, 0|1) records an event (asynchronously);
 * rx_timer_elapsed synchronises and returns the device time between mark 0 and mark 1 in ms.                 */
RX_API int rx_timer_mark(rx_engine *h, int32_t which);
RX_API int rx_timer_elapsed(rx_engine *h, double *ms);
/* Mixing-kernel statistics of the last swap-all call: [0] speculation rounds, [1] exact-path fallbacks,
 * [2] passes, [3] MT words consumed, [4] walker kernel time (us), [5] host wait for the side-stream pre-pass (us). */
RX_API int rx_get_mix_stats(rx_engine *h, int64_t out[6]);
/* Diagnostic: y[t] = the device's correctly rounded exp(x[t]) (host arrays) -- the function behind the one decision the
 * mixing kernels do not take in the log domain, `rand() < exp(log_p)` of replicaexchange.py:340 inside the 1e-9 guard band. */
RX_API int rx_selftest_exp(rx_engine *h, const double *x, double *y, int32_t n);

/* Diagnostic: the launch rx_propagate would make for a RX_SYSTEM_LJ_ALCH or RX_SYSTEM_HARMONIC engine, computed on the host
 * without any device call (so it can be checked without a GPU).  The device enters through n_sm and smem_optin
 * (cudaDevAttrMultiProcessorCount, cudaDevAttrMaxSharedMemoryPerBlockOptin); the environment overrides rx_propagate reads
 * (RX_CLUSTER, RX_SKIN, RX_SKIN_IN, RX_NO_VERLET, RX_NO_SORT) enter through the query.  Returns RX_ERR_UNSUPPORTED for
 * sizes rx_propagate refuses (more than 4096 LJ atoms or 1024 harmonic atoms per replica); the message is then
 * rx_last_error(NULL). */
typedef struct {
    int32_t system_kind, n_atoms;
    int32_t kloc;              /* replicas owned by the engine */
    int32_t per_state;         /* 1: per-state moves (rx_set_state_integrator) are set */
    int32_t n_sm, smem_optin;  /* multiprocessors; opt-in shared memory per block (bytes) */
    double box[3], r_cutoff;
    double skin_out, skin_in;  /* neighbour-list skins (nm); < 0: the defaults 0.40 / 0.05 */
    int32_t cluster;           /* blocks per replica requested (RX_CLUSTER), 0: the planner's choice */
    int32_t no_list, no_sort;  /* all-pairs forces only (RX_NO_VERLET); atoms kept on their threads (RX_NO_SORT) */
} rx_propagate_query;
typedef struct {
    int32_t cluster;           /* thread blocks per replica (a thread-block cluster of 1, 2, 4 or 8) */
    int32_t threads;           /* threads per block, one atom each */
    int32_t list_capacity;     /* neighbour-list entries per atom, 0: all-pairs forces */
    int32_t sort_atoms;        /* 1: atoms are re-dealt to threads by neighbour count at every list build */
    int32_t compact;           /* 1: the layout of more than 1024 atoms (position buffers strided by N, 8-byte parameters) */
    int32_t reserved;
    int64_t smem_bytes;        /* dynamic shared memory per block */
} rx_propagate_plan;
RX_API int rx_plan_propagate(const rx_propagate_query *query, rx_propagate_plan *plan);

/* ---- constant pressure (RX_SYSTEM_LJ_ALCH) -------------------------------------------------------- */
/* Replaces the MonteCarloBarostat that ThermodynamicState(system, temperature, pressure) adds (states.py:1761-1771):
 * isotropic, at the temperature of the replica's state, one attempt every 25 steps (OpenMM's default frequency) inside
 * rx_propagate.  An attempt draws dV uniform in +-volume_scale, scales positions about the origin by (V'/V)^(1/3)
 * (every atom is its own molecule; velocities are not scaled) and accepts when w = dU + p dV - N kT ln(V'/V) <= 0 or
 * u < exp(-w/kT); dU includes the change of the dispersion correction c_l / V.  volume_scale starts at 0.01 V and is
 * divided by 1.1 (acceptance < 25 %) or multiplied by 1.1 up to 0.3 V (acceptance > 75 %) after every 10 attempts.
 * A proposal with a box edge below twice the cutoff is rejected (and counted as an attempt).
 *
 * rx_set_pressures  switches the engine to NPT: pressure[M] in kJ/mol/nm^3 (1 bar = 0.0602214076 kJ/mol/nm^3) and the
 *                   per-state dispersion-correction coefficients dispersion[M] in kJ/mol nm^3 (the correction at volume V
 *                   is dispersion[l] / V; energy_offset of rx_set_states then holds the rest of the offset).  Every owned
 *                   replica gets the box of rx_config and a fresh barostat state.  The energy matrix becomes
 *                   u[k][l] = beta_l (U_l(x_k) + dispersion[l] / V_k + pressure[l] V_k) (states.py:1909-1917).
 * rx_set_boxes / rx_get_boxes  edges[count][3] (nm) of replicas [first, first + count) (global indices, the owned ones).
 * rx_set_barostat / rx_get_barostat  the barostat state of the same replicas (checkpoints); rx_set_boxes leaves it.
 * rx_compute_energies_at_npt  rx_compute_energies_at for an NPT engine: the other states' pressures and dispersion
 *                   coefficients [n] come with them (rx_compute_energies_at returns RX_ERR_INVALID on an NPT engine).
 * rx_minimize minimises every replica at its own box. */
typedef struct {
    double volume_scale;       /* nm^3 */
    int32_t step;              /* steps since the last attempt */
    int32_t n_attempted, n_accepted;   /* since the last adaptation of volume_scale */
    int32_t reserved;
} rx_barostat_state;
RX_API int rx_set_pressures(rx_engine *h, const double *pressure /*[M]*/, const double *dispersion /*[M]*/);
RX_API int rx_set_boxes(rx_engine *h, int32_t first, int32_t count, const double *edges);
RX_API int rx_get_boxes(rx_engine *h, int32_t first, int32_t count, double *edges);
RX_API int rx_set_barostat(rx_engine *h, int32_t first, int32_t count, const rx_barostat_state *state);
RX_API int rx_get_barostat(rx_engine *h, int32_t first, int32_t count, rx_barostat_state *state);
RX_API int rx_compute_energies_at_npt(rx_engine *h, const rx_state_params *states, const double *pressure,
                                      const double *dispersion, int32_t n, double *u_out);
/* rx_compute_energies_at (pressure = dispersion = NULL) or rx_compute_energies_at_npt with the second alchemical region's
 * lambda_sterics [n] of those states (rx_set_alchemical_regions, rx_set_states_region2). */
RX_API int rx_compute_energies_at_region2(rx_engine *h, const rx_state_params *states, const double *lambda_sterics_2,
                                          const double *pressure, const double *dispersion, int32_t n, double *u_out);

/* ---- multi-GPU ------------------------------------------------------------------------------------ */
/* NCCL is loaded with dlopen(nccl_library_path).  Rank 0 creates an id (rx_comm_unique_id), the host code
 * distributes its bytes (torch.distributed / MPI / a file), every rank calls rx_comm_init.  Replaces
 * mpiplus.distribute(..., send_results_to=0) (multistatesampler.py:1296,1448).                             */
RX_API int rx_comm_unique_id(const char *nccl_library_path, void *id_out /*128 bytes*/);
RX_API int rx_comm_init(rx_engine *h, const char *nccl_library_path, const void *unique_id /*128 bytes*/);

#ifdef __cplusplus
}
#endif
#endif /* RX_B200_H */
