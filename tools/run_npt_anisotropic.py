"""Cost of the anisotropic barostat on the headline system: the alchemical LJ fluid (512 atoms, 500 steps per iteration,
swap-all) at constant pressure with the isotropic barostat, the anisotropic one scaling x, y and z, and the anisotropic
one scaling z alone, alternated in one process.  One attempt costs the same in all three (two energy sums, two list
rebuilds), so their propagation times should agree within noise.

  run_npt_anisotropic.py time [--K 256] [--iterations 20] [--rounds 3] [--pressure-bar 50]
      one JSON line per (K, barostat, round): iterations/s of the fused device loop (rx_run_iterations), propagation ms per
      iteration (device events), acceptance and mean volume, with the GPU's name and power limit.
  run_npt_anisotropic.py digest [--K 64] [--iterations 6]
      one JSON line: SHA-256 digests of positions, velocities, boxes and barostat records after an isotropic NPT run of the
      fused loop, for the library in use (RX_B200_LIB selects another build).
  run_npt_anisotropic.py ab LIB_A[@TREE_A] LIB_B[@TREE_B] [--K 64] [--iterations 6]
      `digest` in one child process per library, with the Python package of TREE (default: this tree), so that a build
      of another commit runs with its own bindings; exits 1 unless every digest agrees."""
import argparse, hashlib, json, os, subprocess, sys, time
import numpy as np
ROOT = os.environ.get('NPT_DIGEST_TREE') or os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from openmmtools_b200 import alchemy, mcmc, multistate, states, unit

BAROSTATS = {'isotropic': None, 'anisotropic-xyz': (True, True, True), 'anisotropic-z': (False, False, True)}


def sampler(K, pressure_bar, scale):
    fluid, asys, tstates, sstate, lambdas = bench.build_workload(K, 512)
    if scale is None:
        for t in tstates:
            t.pressure = pressure_bar * unit.bar
    else:
        from openmmtools_b200.system import MonteCarloAnisotropicBarostat
        asys = asys.copy()
        asys.addForce(MonteCarloAnisotropicBarostat(pressure_bar * unit.bar, 300.0 * unit.kelvin, *scale))
        tstates = states.create_thermodynamic_state_protocol(
            asys, {'lambda_sterics': lambdas, 'lambda_electrostatics': lambdas}, constants={'temperature': 300.0 * unit.kelvin},
            composable_states=alchemy.AlchemicalState.from_system(asys))
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, collision_rate=10.0 / unit.picosecond, n_steps=500,
                                              splitting='V R O R V', reassign_velocities=False)
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=10 ** 9, replica_mixing_scheme='swap-all', seed=1234)
    s.create(tstates, [sstate], storage=None)
    s._compute_energies()
    return s


def gpu_and_power():
    import torch
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True,
                               text=True).stdout.strip()
    except OSError:
        power = 'unknown'
    return torch.cuda.get_device_name(0), power


def time_barostats(a):
    gpu, power = gpu_and_power()
    for K in a.K:
        runs = {name: sampler(K, a.pressure_bar, scale) for name, scale in BAROSTATS.items()}
        it = {m: 1 for m in runs}
        for m, s in runs.items():      # warm-up: module loads, first list builds, step-size adaptation
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
                b = e.get_barostat() if BAROSTATS[m] is None else e.get_barostat_anisotropic()
                acc = float(b['n_accepted'].sum() / max(b['n_attempted'].sum(), 1))
                print(json.dumps(dict(K=K, barostat=m, round=r, iterations_per_s=a.iterations / dt,
                                      propagate_ms_per_iteration=pt['propagate_ms'] / a.iterations,
                                      energies_ms_per_iteration=pt['energies_ms'] / a.iterations,
                                      barostat_acceptance=acc, mean_volume_nm3=float(np.prod(e.get_boxes(), axis=1).mean()),
                                      gpu=gpu, power_limit=power)), flush=True)


def digest(a):
    s = sampler(a.K[0], a.pressure_bar, None)
    e = s._engine
    e.run_iterations(a.iterations, 'swap-all', s._seed, 1)
    b = e.get_barostat()
    parts = dict(positions=e.get_positions(), velocities=e.get_velocities(), boxes=e.get_boxes(),
                 barostat=np.stack([b['volume_scale'], b['step'], b['n_attempted'], b['n_accepted']]),
                 replica_states=e.get_replica_states())
    out = {k: hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest()[:16] for k, v in parts.items()}
    out.update(library=os.environ.get('RX_B200_LIB', 'default'), tree=ROOT, K=a.K[0], iterations=a.iterations)
    print(json.dumps(out), flush=True)


def ab(a):
    results = []
    for spec in a.libs:
        lib, _, tree = spec.partition('@')
        env = dict(os.environ, RX_B200_LIB=os.path.abspath(lib))
        if tree:
            env['NPT_DIGEST_TREE'] = os.path.abspath(tree)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), 'digest', '--K', str(a.K[0]), '--iterations',
                            str(a.iterations)], env=env, capture_output=True, text=True)
        if r.returncode:
            sys.exit(r.stdout + r.stderr)
        line = r.stdout.strip().splitlines()[-1]
        print(line, flush=True)
        results.append({k: v for k, v in json.loads(line).items() if k not in ('library', 'tree')})
    same = all(r == results[0] for r in results)
    print(json.dumps(dict(identical=same)), flush=True)
    sys.exit(0 if same else 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('mode', choices=['time', 'digest', 'ab'])
    ap.add_argument('libs', nargs='*')
    ap.add_argument('--K', type=int, nargs='+', default=None)
    ap.add_argument('--iterations', type=int, default=None)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--pressure-bar', type=float, default=50.0)
    a = ap.parse_args()
    if a.K is None:
        a.K = [256] if a.mode == 'time' else [64]
    if a.iterations is None:
        a.iterations = 20 if a.mode == 'time' else 6
    {'time': time_barostats, 'digest': digest, 'ab': ab}[a.mode](a)


if __name__ == '__main__':
    main()
