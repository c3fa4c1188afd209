"""Launch plan of k_propagate (rx_plan_propagate: host arithmetic, no device).  Up to 1024 atoms it must equal the plan
the engine has always made; from 1025 to 4096 atoms every plan must fit an H100 block and keep a neighbour list of at
least 48 entries per atom at LennardJonesFluid's default parameters (DESIGN 4.2)."""
import numpy as np
import pytest
from openmmtools_b200._engine import Engine, EngineError
from openmmtools_b200._lib import RX_SYSTEM_LJ_ALCH, RX_SYSTEM_HARMONIC, RX_ERR_UNSUPPORTED
from helpers import SIGMA

N_SM, OPTIN = 132, 227 * 1024        # H100 SXM: multiprocessors, opt-in shared memory per block
RC = 3.0 * SIGMA
KLOCS = (1, 8, 33, 64, 256)


def fluid_box(N, reduced_density=0.05):
    """Cubic box edge of LennardJonesFluid(nparticles=N) at its default density."""
    return (N * SIGMA ** 3 / reduced_density) ** (1.0 / 3.0)


def plan(N, kloc, kind=RX_SYSTEM_LJ_ALCH, per_state=False, no_list=False, L=None, **kw):
    L = fluid_box(N) if L is None else L
    return Engine.plan_propagate(kind, N, kloc, kw.pop('n_sm', N_SM), kw.pop('smem_optin', OPTIN), box=(L, L, L),
                                 r_cutoff=RC, per_state=per_state, no_list=no_list, **kw)


def plan_up_to_1024(N, kloc, per_state, no_list, L, lj=True):
    """The launch rxi_propagate made for N <= 1024 before replicas could exceed 1024 atoms, restated."""
    cl = 4 if lj and N >= 256 and kloc * 4 <= N_SM else 1
    if per_state:
        cl = 1
    threads = -(-(-(-N // cl)) // 32) * 32
    atoms_bytes = 3 * 1024 * 16 + threads * 16
    area, cap, sort = threads * 16, 0, False
    if lj and N >= 64 and not no_list:
        rl = min(RC + 0.40, 0.5 * L)
        eff_out = rl - RC
        if eff_out > 0.03:
            budget = (200 if threads > 512 else 112) * 1024
            c = min((budget - atoms_bytes) // (threads * 2), 128)
            if c >= 8:
                cap = c
                list_bytes = (c * threads * 2 + 15) // 16 * 16
                sort = list_bytes >= threads * 18 + (threads // 32 + 1) * 128 * 2
                area = max(area, list_bytes)
    return dict(cluster=cl, threads=threads, list_capacity=cap, sort_atoms=sort, compact=False, smem_bytes=atoms_bytes + area)


@pytest.mark.parametrize('kloc', KLOCS)
@pytest.mark.parametrize('per_state', [False, True])
@pytest.mark.parametrize('no_list', [False, True])
def test_plan_up_to_1024_atoms_is_unchanged(kloc, per_state, no_list):
    for N in range(1, 1025):
        L = fluid_box(N)
        assert plan(N, kloc, per_state=per_state, no_list=no_list) == plan_up_to_1024(N, kloc, per_state, no_list, L), N


def test_harmonic_plan_up_to_1024_atoms_is_unchanged():
    for N in (1, 31, 256, 1000, 1024):
        for kloc in KLOCS:
            assert plan(N, kloc, kind=RX_SYSTEM_HARMONIC) == plan_up_to_1024(N, kloc, False, True, fluid_box(N), lj=False)


def test_cluster_pin_up_to_1024_atoms_accepts_1_2_4_only():
    for cl in (1, 2, 4):
        assert plan(777, 64, cluster=cl)['cluster'] == cl
    assert plan(777, 64, cluster=8)['cluster'] == 1         # ignored, as before
    assert plan(200, 1, cluster=4)['cluster'] == 1          # (below 256 atoms one block, pinned or not)


@pytest.mark.parametrize('kloc', KLOCS)
@pytest.mark.parametrize('per_state', [False, True])
def test_plan_from_1025_to_4096_atoms_fits_and_keeps_a_list(kloc, per_state):
    for N in range(1025, 4097):
        p = plan(N, kloc, per_state=per_state)
        assert p['compact'] and p['cluster'] in (2, 4, 8), (N, p)
        assert p['threads'] <= 1024 and p['threads'] * p['cluster'] >= N and p['threads'] % 32 == 0, (N, p)
        assert p['smem_bytes'] <= OPTIN, (N, p)
        assert p['list_capacity'] >= 48, (N, p)
        # atoms: two position buffers (16 B), parameters (8 B); per thread a reference position and the list column
        assert p['smem_bytes'] >= 40 * N + p['threads'] * (16 + 2 * p['list_capacity']), (N, p)


def test_cluster_choice_above_1024_atoms():
    # the smallest cluster that holds the atoms with a list of 48 entries, widened while kloc * CL <= #SMs
    assert plan(2048, 64)['cluster'] == 2 and plan(2048, 34)['cluster'] == 2
    assert plan(2048, 16)['cluster'] == 8 and plan(2048, 33)['cluster'] == 4
    assert plan(3000, 64)['cluster'] == 4
    assert plan(4096, 64)['cluster'] == 8 and plan(4096, 256)['cluster'] == 8
    # RX_CLUSTER is honoured where that cluster holds the atoms and a list, ignored otherwise
    assert [plan(2048, 64, cluster=c)['cluster'] for c in (1, 2, 4, 8)] == [2, 2, 4, 8]
    assert [plan(4096, 64, cluster=c)['cluster'] for c in (2, 4, 8)] == [8, 8, 8]
    assert [plan(1025, 256, cluster=c)['cluster'] for c in (2, 4, 8)] == [2, 4, 8]
    # all-pairs forces (no list): the smallest cluster that holds the atoms
    p = plan(4096, 256, no_list=True)
    assert p['cluster'] == 4 and p['list_capacity'] == 0 and p['threads'] == 1024


def test_sizes_beyond_the_kernels_are_refused():
    for kind, N in ((RX_SYSTEM_LJ_ALCH, 4097), (RX_SYSTEM_HARMONIC, 1025)):
        with pytest.raises(EngineError) as e:
            plan(N, 1, kind=kind)
        assert e.value.code == RX_ERR_UNSUPPORTED and 'not supported' in e.value.message
    # a device with less shared memory than the atoms need
    with pytest.raises(EngineError) as e:
        plan(4096, 1, smem_optin=100 * 1024)
    assert e.value.code == RX_ERR_UNSUPPORTED and 'do not fit' in e.value.message
