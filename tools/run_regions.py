"""Cost of a second alchemical region on the headline shape: 256 replicas of the 512-atom alchemical LJ fluid, 500
steps per iteration, swap-all; one region of 5 atoms against two regions of 5 atoms each (a dual-topology ladder,
lambda_B = 1 - lambda_A), alternated in one process.

Prints one JSON line per (regions, round): iterations/s of the fused device loop (rx_run_iterations) and the mix,
propagate and energy phases per iteration (device events), with the card's name and power limit.
usage: run_regions.py [--K 256] [--iterations 10] [--rounds 3]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openmmtools_b200 import testsystems, alchemy, states, mcmc, multistate, unit


def sampler(K, two):
    fluid = testsystems.LennardJonesFluid(nparticles=512)
    factory = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True)
    lam = [1.0 - l / (K - 1) for l in range(K)]
    if two:
        regions = [alchemy.AlchemicalRegion(alchemical_atoms=range(5), name='A'),
                   alchemy.AlchemicalRegion(alchemical_atoms=range(5, 10), name='B')]
        asys = factory.create_alchemical_system(fluid.system, regions)
        comp = [alchemy.AlchemicalState.from_system(asys, parameters_name_suffix=n) for n in ('A', 'B')]
        protocol = {'lambda_sterics_A': lam, 'lambda_sterics_B': [1.0 - v for v in lam]}
    else:
        asys = factory.create_alchemical_system(fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(5)))
        comp = [alchemy.AlchemicalState.from_system(asys)]
        protocol = {'lambda_sterics': lam}
    tstates = states.create_thermodynamic_state_protocol(asys, protocol, constants={'temperature': 300.0 * unit.kelvin},
                                                         composable_states=comp)
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, collision_rate=10.0 / unit.picosecond, n_steps=500,
                                              splitting='V R O R V', reassign_velocities=False)
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=10 ** 9, replica_mixing_scheme='swap-all', seed=1234)
    s.create(tstates, [sstate], storage=None)
    s._compute_energies()
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--K', type=int, default=256)
    ap.add_argument('--iterations', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    import torch
    gpu = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True,
                               text=True).stdout.strip()
    except OSError:
        power = 'unknown'
    runs = {1: sampler(a.K, False), 2: sampler(a.K, True)}
    it = {m: 1 for m in runs}
    for m, s in runs.items():      # warm-up: module loads, first list builds
        s._engine.run_iterations(3, 'swap-all', s._seed, it[m])
        it[m] += 3
    for r in range(a.rounds):
        for m, s in runs.items():
            e = s._engine
            e.phase_times(reset=True)
            t0 = time.perf_counter()
            e.run_iterations(a.iterations, 'swap-all', s._seed, it[m])
            dt = time.perf_counter() - t0
            it[m] += a.iterations
            pt = e.phase_times()
            print(json.dumps(dict(K=a.K, N=512, regions=m, round=r, iterations_per_s=a.iterations / dt,
                                  mix_ms_per_iteration=pt['mix_ms'] / a.iterations,
                                  propagate_ms_per_iteration=pt['propagate_ms'] / a.iterations,
                                  energies_ms_per_iteration=pt['energies_ms'] / a.iterations, gpu=gpu, power_limit=power)),
                  flush=True)


if __name__ == '__main__':
    main()
