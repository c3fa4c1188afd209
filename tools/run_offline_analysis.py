"""Time one offline free-energy pass two ways, one JSON line per size (K replicas = K states, T iterations):

- from the device history: the sampler's pass (the effective-energy timeseries and equilibration on the K doubles per
  iteration the sampler keeps on the host, u_kn gathered on the device from the engine's energy history, MBAR);
- from storage: MultiStateSamplerAnalyzer on the stored run, the way the reference's pass works (read every stored
  energy matrix, lay u_kn out on the host, upload it, MBAR).

Both start MBAR from zeros and give the same free energy.  The energies are synthetic (uncorrelated, one state offset
per state, a random permutation of the states per iteration).  Storage goes to a temporary directory.

    python tools/run_offline_analysis.py [--sizes 64x5000,256x2000,256x10000]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from openmmtools_b200 import _lib, multistate
from openmmtools_b200._engine import Engine
from openmmtools_b200.multistate.mbar import MBAR
from openmmtools_b200.multistate.multistateanalyzer import (decorrelated_iterations, effective_energy_timeseries,
                                                            equilibration_data)


def _gpu():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def _synchronize():
    import torch
    torch.cuda.synchronize()


def one(K, T, tmp, seed=0):
    rng = np.random.default_rng(seed)
    offset = 0.05 * np.arange(K)
    e = Engine(0, K, K)
    path = os.path.join(tmp, 'run')
    r = multistate.MultiStateReporter(path, open_mode='w')
    r.set_dimensions(K, K, 1)
    r.write_thermodynamic_states([], [])
    u_kept, s_kept = [], []
    nb = np.ones((K, K), np.int8)
    for t in range(T + 1):
        u = rng.standard_normal((K, K)) + offset[None, :]
        st = rng.permutation(K)
        e.set_energies(u)
        e.history_append(t)
        r.write_energies(u, nb, np.zeros((K, 0)), t)
        r.write_replica_thermodynamic_states(st, t)
        r.write_last_iteration(t)
        u_kept.append(u[np.arange(K), st])
        s_kept.append(st)
    r.close()
    os.sync()

    # -- from the device history
    _synchronize()
    t0 = time.perf_counter()
    states = np.stack(s_kept, axis=1)
    u_n = effective_energy_timeseries(np.stack(u_kept, axis=1), states)
    n_eq, g, _ = equilibration_data(u_n, 1, 100)
    selected = decorrelated_iterations(n_eq, g, T)
    N_k = np.zeros(K, np.int64)
    v, c = np.unique(states[:, selected], return_counts=True)
    N_k[v] = c
    t1 = time.perf_counter()
    lib = _lib.load()
    h = C.c_void_p()
    it = np.ascontiguousarray(selected, dtype=np.int64)
    cols = np.arange(K, dtype=np.int32)
    assert lib.rx_mbar_create_from_history(e._h, K, len(it), it.ctypes.data_as(C.c_void_p), cols.ctypes.data_as(C.c_void_p),
                                           N_k.ctypes.data_as(C.c_void_p), C.byref(h)) == 0
    t2 = time.perf_counter()
    lib.rx_mbar_destroy(h)
    t3 = time.perf_counter()
    m = MBAR.from_history(e, selected, cols, N_k, initial_f_k=np.zeros(K))
    dev = m.compute_free_energy_differences()
    m.close()
    t4 = time.perf_counter()
    device = {'pass_s': (t1 - t0) + (t4 - t3), 'host_timeseries_s': t1 - t0, 'gather_create_s': t2 - t1,
              'mbar_iterations': m.n_iterations}

    # -- from storage (MultiStateSamplerAnalyzer, the reference's pass)
    t0 = time.perf_counter()
    a = multistate.MultiStateSamplerAnalyzer(multistate.MultiStateReporter(path, open_mode='r'),
                                             analysis_kwargs={'initial_f_k': np.zeros(K)})
    a._decorrelated
    t1 = time.perf_counter()
    D, dD = a.get_free_energy()
    t2 = time.perf_counter()
    storage = {'pass_s': t2 - t0, 'read_and_layout_s': t1 - t0}
    same = bool(D[0, -1] == dev['Delta_f'][0, -1] and dD[0, -1] == dev['dDelta_f'][0, -1])
    e.close()
    return {'K': K, 'T': T, 'n_samples': int(K * len(selected)), 'device_history': device, 'storage': storage,
            'speedup': storage['pass_s'] / device['pass_s'], 'same_free_energy': same,
            'history_bytes': int(8 * K * K * (T + 1)), 'gpu': _gpu()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--sizes', default='64x5000,256x2000,256x10000')
    p.add_argument('--tmp', default=None, help='directory for the stored runs (default: a temporary directory)')
    args = p.parse_args()
    for size in args.sizes.split(','):
        K, T = (int(x) for x in size.split('x'))
        tmp = tempfile.mkdtemp(dir=args.tmp)
        try:
            print(json.dumps(one(K, T, tmp)), flush=True)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
