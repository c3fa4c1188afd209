"""ctypes binding of librx_b200.so (include/rx_b200.h).

There is NO CPU fallback: if the shared library is missing or no CUDA device is visible, engine creation
raises.  (The CPU oracle under /oracle is test infrastructure and is never imported from here.)
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('RX_B200_LIB') or os.path.join(_HERE, 'csrc', 'librx_b200.so')   # override: A/B builds

RX_ABI_VERSION = 1
RX_OK, RX_ERR_INVALID, RX_ERR_CUDA, RX_ERR_NAN, RX_ERR_UNSUPPORTED, RX_ERR_COMM, RX_ERR_CAPACITY = 0, -1, -2, -3, -4, -5, -6
RX_SYSTEM_NONE, RX_SYSTEM_LJ_ALCH, RX_SYSTEM_HARMONIC, RX_SYSTEM_MOLECULE = 0, 1, 2, 3
RX_STREAM_NUMBA, RX_STREAM_NUMPY = 0, 1

# every symbol include/rx_b200.h declares
SYMBOLS = [
    'rx_create', 'rx_destroy', 'rx_last_error', 'rx_abi_version', 'rx_set_particles', 'rx_set_states',
    'rx_set_integrator', 'rx_set_state_integrator', 'rx_set_molecule', 'rx_set_implicit_solvent', 'rx_set_positions', 'rx_set_velocities', 'rx_get_positions', 'rx_get_velocities',
    'rx_get_replica_energies', 'rx_pin_host_memory', 'rx_unpin_host_memory', 'rx_randomize_velocities', 'rx_minimize', 'rx_set_replica_states', 'rx_get_replica_states',
    'rx_propagate', 'rx_propagate_retry', 'rx_compute_energies', 'rx_compute_energies_at', 'rx_set_energies', 'rx_get_energies', 'rx_mix_seed',
    'rx_mix_skip', 'rx_mix_swap_all', 'rx_mix_swap_neighbors', 'rx_get_mix_counts', 'rx_mix_stream_position',
    'rx_run_iterations', 'rx_sams_set', 'rx_sams_step', 'rx_sams_get', 'rx_sams_run_iterations', 'rx_get_phase_times', 'rx_timer_mark', 'rx_timer_elapsed', 'rx_get_mix_stats', 'rx_selftest_exp', 'rx_plan_propagate', 'rx_comm_unique_id', 'rx_comm_init',
    'rx_set_pressures', 'rx_set_boxes', 'rx_get_boxes', 'rx_set_barostat', 'rx_get_barostat', 'rx_compute_energies_at_npt',
    'rx_set_alchemical_regions', 'rx_set_states_region2', 'rx_compute_energies_at_region2',
    'rx_set_mc_subsets', 'rx_set_state_mc_moves', 'rx_get_mc_statistics', 'rx_set_mc_statistics', 'rx_get_mc_energy_changes',
]
RX_MAX_MC_MOVES = 4
RX_MC_DISPLACEMENT, RX_MC_ROTATION = 0, 1


class RxConfig(C.Structure):
    _fields_ = [('abi_version', C.c_int32), ('system_kind', C.c_int32), ('n_replicas', C.c_int32),
                ('n_states', C.c_int32), ('n_atoms', C.c_int32), ('device', C.c_int32), ('rank', C.c_int32),
                ('world_size', C.c_int32), ('box', C.c_double * 3), ('r_cutoff', C.c_double),
                ('r_switch', C.c_double), ('use_switch', C.c_int32), ('annihilate_sterics', C.c_int32),
                ('softcore_alpha', C.c_double), ('softcore_a', C.c_double), ('softcore_b', C.c_double),
                ('softcore_c', C.c_double)]


class RxStateParams(C.Structure):
    _fields_ = [('temperature', C.c_double), ('lambda_sterics', C.c_double), ('energy_offset', C.c_double),
                ('ho_K', C.c_double), ('ho_x0', C.c_double * 3)]


class RxSamsConfig(C.Structure):
    _fields_ = [('gamma0', C.c_double), ('flatness_threshold', C.c_double), ('weight_update_method', C.c_int32),
                ('two_stage', C.c_int32), ('flatness_criteria', C.c_int32), ('stage', C.c_int32), ('t0', C.c_int64)]


class RxPropagateQuery(C.Structure):
    _fields_ = [('system_kind', C.c_int32), ('n_atoms', C.c_int32), ('kloc', C.c_int32), ('per_state', C.c_int32),
                ('n_sm', C.c_int32), ('smem_optin', C.c_int32), ('box', C.c_double * 3), ('r_cutoff', C.c_double),
                ('skin_out', C.c_double), ('skin_in', C.c_double), ('cluster', C.c_int32), ('no_list', C.c_int32),
                ('no_sort', C.c_int32)]


class RxPropagatePlan(C.Structure):
    _fields_ = [('cluster', C.c_int32), ('threads', C.c_int32), ('list_capacity', C.c_int32), ('sort_atoms', C.c_int32),
                ('compact', C.c_int32), ('reserved', C.c_int32), ('smem_bytes', C.c_int64)]


class RxBarostatState(C.Structure):
    _fields_ = [('volume_scale', C.c_double), ('step', C.c_int32), ('n_attempted', C.c_int32), ('n_accepted', C.c_int32),
                ('reserved', C.c_int32)]


class RxMolecule(C.Structure):
    _fields_ = [('n_bonds', C.c_int32), ('n_angles', C.c_int32), ('n_torsions', C.c_int32), ('n_exclusions', C.c_int32),
                ('n_exceptions', C.c_int32), ('n_constraints', C.c_int32), ('remove_cm_motion', C.c_int32), ('reserved', C.c_int32),
                ('constraint_tolerance', C.c_double),
                ('mass', C.c_void_p), ('charge', C.c_void_p), ('sigma', C.c_void_p), ('epsilon', C.c_void_p),
                ('bonds', C.c_void_p), ('angles', C.c_void_p), ('torsions', C.c_void_p), ('exclusions', C.c_void_p),
                ('exceptions', C.c_void_p), ('constraints', C.c_void_p)]


class RxMcMove(C.Structure):
    _fields_ = [('kind', C.c_int32), ('subset_offset', C.c_int32), ('subset_len', C.c_int32), ('reserved', C.c_int32),
                ('sigma_nm', C.c_double)]


class RxGbsa(C.Structure):
    _fields_ = [('radius', C.c_void_p), ('scale', C.c_void_p), ('alpha', C.c_double), ('beta', C.c_double), ('gamma', C.c_double),
                ('offset', C.c_double), ('solute_dielectric', C.c_double), ('solvent_dielectric', C.c_double),
                ('sa_energy', C.c_double), ('probe_radius', C.c_double)]


_lib = None


def load():
    """Load librx_b200.so; raises ImportError with build instructions if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            'openmmtools_b200: the CUDA extension %s has not been built (run `python -c "import __graft_entry__ as g; '
            'g.build()"` or `make -C openmmtools_b200/csrc`). There is no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, u64, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_double
    lib.rx_last_error.restype = C.c_char_p
    lib.rx_last_error.argtypes = [vp]
    lib.rx_create.argtypes = [C.POINTER(RxConfig), C.POINTER(vp)]
    lib.rx_destroy.argtypes = [vp]
    lib.rx_destroy.restype = None
    lib.rx_set_particles.argtypes = [vp, vp, vp, vp, vp]
    lib.rx_set_states.argtypes = [vp, vp]
    lib.rx_set_integrator.argtypes = [vp, dbl, dbl, i32, C.c_char_p]
    lib.rx_set_state_integrator.argtypes = [vp, i32, dbl, dbl, i32, C.c_char_p, i32]
    lib.rx_set_molecule.argtypes = [vp, C.POINTER(RxMolecule)]
    lib.rx_set_implicit_solvent.argtypes = [vp, C.POINTER(RxGbsa)]
    for name in ('rx_set_positions', 'rx_set_velocities', 'rx_get_positions', 'rx_get_velocities'):
        getattr(lib, name).argtypes = [vp, i32, i32, vp]
    lib.rx_get_replica_energies.argtypes = [vp, vp, vp]
    lib.rx_pin_host_memory.argtypes = [vp, vp, u64]
    lib.rx_unpin_host_memory.argtypes = [vp, vp]
    lib.rx_randomize_velocities.argtypes = [vp, u64, u64]
    lib.rx_minimize.argtypes = [vp, dbl, i32, vp, vp]
    lib.rx_set_replica_states.argtypes = [vp, vp]
    lib.rx_get_replica_states.argtypes = [vp, vp]
    lib.rx_propagate.argtypes = [vp, u64, u64, i32, vp]
    lib.rx_propagate_retry.argtypes = [vp, u64, u64, i32, vp]
    lib.rx_compute_energies.argtypes = [vp, vp]
    lib.rx_compute_energies_at.argtypes = [vp, vp, i32, vp]
    lib.rx_set_energies.argtypes = [vp, vp]
    lib.rx_get_energies.argtypes = [vp, vp]
    lib.rx_mix_seed.argtypes = [vp, i32, C.c_uint32]
    lib.rx_mix_skip.argtypes = [vp, i32, u64]
    lib.rx_mix_swap_all.argtypes = [vp, i64, vp, vp, vp]
    lib.rx_mix_swap_neighbors.argtypes = [vp, vp, vp, vp]
    lib.rx_get_mix_counts.argtypes = [vp, vp, vp]
    lib.rx_mix_stream_position.argtypes = [vp, i32, C.POINTER(u64)]
    lib.rx_run_iterations.argtypes = [vp, i32, i32, u64, u64, i32]
    lib.rx_sams_set.argtypes = [vp, C.POINTER(RxSamsConfig), vp, vp, vp]
    lib.rx_sams_step.argtypes = [vp, i64, i32, vp]
    lib.rx_sams_get.argtypes = [vp, vp, vp, vp, C.POINTER(i32), C.POINTER(i64), C.POINTER(dbl), vp, vp]
    lib.rx_sams_run_iterations.argtypes = [vp, i32, u64, u64, i32]
    lib.rx_get_phase_times.argtypes = [vp, vp, vp, i32]
    lib.rx_timer_mark.argtypes = [vp, i32]
    lib.rx_timer_elapsed.argtypes = [vp, C.POINTER(dbl)]
    lib.rx_get_mix_stats.argtypes = [vp, vp]
    lib.rx_selftest_exp.argtypes = [vp, vp, vp, C.c_int32]
    lib.rx_plan_propagate.argtypes = [C.POINTER(RxPropagateQuery), C.POINTER(RxPropagatePlan)]
    lib.rx_comm_unique_id.argtypes = [C.c_char_p, vp]
    lib.rx_comm_init.argtypes = [vp, C.c_char_p, vp]
    lib.rx_set_pressures.argtypes = [vp, vp, vp]
    lib.rx_compute_energies_at_npt.argtypes = [vp, vp, vp, vp, i32, vp]
    lib.rx_set_alchemical_regions.argtypes = [vp, vp, i32, i32]
    lib.rx_set_states_region2.argtypes = [vp, vp]
    lib.rx_compute_energies_at_region2.argtypes = [vp, vp, vp, vp, vp, i32, vp]
    lib.rx_set_mc_subsets.argtypes = [vp, vp, i32]
    lib.rx_set_state_mc_moves.argtypes = [vp, i32, i32, vp]
    lib.rx_get_mc_statistics.argtypes = [vp, vp, vp]
    lib.rx_set_mc_statistics.argtypes = [vp, vp, vp]
    lib.rx_get_mc_energy_changes.argtypes = [vp, vp]
    for name in ('rx_set_boxes', 'rx_get_boxes', 'rx_set_barostat', 'rx_get_barostat'):
        getattr(lib, name).argtypes = [vp, i32, i32, vp]
    if lib.rx_abi_version() != RX_ABI_VERSION:
        raise ImportError('librx_b200.so ABI version mismatch')
    _lib = lib
    return lib


def find_nccl():
    """Path of a libnccl.so.2 for dlopen (multi-GPU only)."""
    cands = []
    try:
        import importlib.util
        spec = importlib.util.find_spec('nvidia.nccl')
        if spec and spec.submodule_search_locations:
            for p in spec.submodule_search_locations:
                cands.append(os.path.join(p, 'lib', 'libnccl.so.2'))
    except Exception:
        pass
    cands += ['/usr/lib/x86_64-linux-gnu/libnccl.so.2', 'libnccl.so.2']
    for c in cands:
        if os.path.sep not in c or os.path.exists(c):
            return c
    return 'libnccl.so.2'
