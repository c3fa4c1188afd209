"""Cost of constant pressure on the headline system: the alchemical LJ fluid (512 atoms, 500 steps per iteration,
swap-all) under NVT and under NPT (a Monte Carlo barostat attempt every 25 steps), alternated in one process.

Prints one JSON line per (K, ensemble, round): iterations/s of the fused device loop (rx_run_iterations), propagation ms
per iteration (device events), and for NPT the barostat's acceptance over the replicas' current adaptation windows.
usage: run_npt.py [--K 64 256] [--iterations 20] [--rounds 3] [--pressure-bar 50]"""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from openmmtools_b200 import mcmc, multistate, unit


def sampler(K, pressure_bar):
    fluid, asys, tstates, sstate, lambdas = bench.build_workload(K, 512)
    if pressure_bar is not None:
        for t in tstates:
            t.pressure = pressure_bar * unit.bar
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, collision_rate=10.0 / unit.picosecond, n_steps=500,
                                              splitting='V R O R V', reassign_velocities=False)
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=10 ** 9, replica_mixing_scheme='swap-all', seed=1234)
    s.create(tstates, [sstate], storage=None)
    s._compute_energies()
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--K', type=int, nargs='+', default=[64, 256])
    ap.add_argument('--iterations', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--pressure-bar', type=float, default=50.0)
    a = ap.parse_args()
    import torch
    gpu = torch.cuda.get_device_name(0)
    try:
        import subprocess
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True,
                               text=True).stdout.strip()
    except OSError:
        power = 'unknown'
    for K in a.K:
        runs = {'NVT': sampler(K, None), 'NPT': sampler(K, a.pressure_bar)}
        it = {m: 1 for m in runs}
        for m, s in runs.items():      # warm-up: module loads, first list builds, barostat adaptation
            s._engine.run_iterations(5, 'swap-all', s._seed, it[m])
            it[m] += 5
        for r in range(a.rounds):
            for m, s in runs.items():
                e = s._engine
                e.phase_times(reset=True)
                t0 = time.perf_counter()
                e.run_iterations(a.iterations, 'swap-all', s._seed, it[m])
                dt = time.perf_counter() - t0
                it[m] += a.iterations
                pt = e.phase_times()
                rec = dict(K=K, ensemble=m, round=r, iterations_per_s=a.iterations / dt,
                           propagate_ms_per_iteration=pt['propagate_ms'] / a.iterations,
                           energies_ms_per_iteration=pt['energies_ms'] / a.iterations, gpu=gpu, power_limit=power)
                if m == 'NPT':
                    b = e.get_barostat()
                    rec['barostat_acceptance'] = float(b['n_accepted'].sum() / max(b['n_attempted'].sum(), 1))
                    rec['mean_volume_nm3'] = float(np.prod(e.get_boxes(), axis=1).mean())
                print(json.dumps(rec), flush=True)


if __name__ == '__main__':
    main()
