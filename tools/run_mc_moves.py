"""Cost of the Monte Carlo rigid-body moves on the headline shape: the 512-atom alchemical LJ fluid (5 alchemical atoms,
the ligand), 500 Langevin steps per iteration, swap-all, at K = 64 and 256 replicas; the Langevin move alone against YANK's
SequenceMove([MCDisplacementMove(ligand), MCRotationMove(ligand), Langevin]), alternated in one process.

Prints one JSON line per (K, moves, round): iterations/s of the fused device loop (rx_run_iterations), and per iteration the
mix and propagate phases (device events; the propagate phase holds the Monte Carlo launches), with the card's name and power
limit; then per (K, moves) one line of kernel times per iteration from a torch.profiler pass of its own: k_mc_move and
k_propagate, so that the Monte Carlo launches and any change of the Langevin kernel itself are told apart.
usage: run_mc_moves.py [--K 64 256] [--iterations 10] [--rounds 3]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openmmtools_b200 import testsystems, alchemy, states, mcmc, multistate, unit

LIGAND = list(range(5))


def sampler(K, mc):
    fluid = testsystems.LennardJonesFluid(nparticles=512)
    asys = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True).create_alchemical_system(
        fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=LIGAND))
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': [1.0 - l / (K - 1) for l in range(K)]}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=alchemy.AlchemicalState.from_system(asys))
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    move = mcmc.LangevinSplittingDynamicsMove(timestep=1.0 * unit.femtosecond, collision_rate=10.0 / unit.picosecond, n_steps=500)
    if mc:
        move = mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.1 * unit.nanometer, atom_subset=LIGAND),
                                  mcmc.MCRotationMove(atom_subset=LIGAND), move])
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=10 ** 9, replica_mixing_scheme='swap-all', seed=1234)
    s.create(tstates, [sstate], storage=None)
    s._compute_energies()
    return s


def kernel_ms(s, first, n):
    """Device time per iteration of the k_mc_move and k_propagate launches of n fused iterations (torch.profiler)."""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s._engine.run_iterations(n, 'swap-all', s._seed, first)
    ms = lambda name: sum(e.device_time_total for e in prof.key_averages()
                          if e.key.removeprefix('void ').startswith(name + '<') or e.key.removeprefix('void ').startswith(name + '(')) / 1e3 / n
    return dict(k_mc_move_ms=ms('k_mc_move'), k_propagate_ms=ms('k_propagate'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--K', type=int, nargs='+', default=[64, 256])
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
    for K in a.K:
        runs = {False: sampler(K, False), True: sampler(K, True)}
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
                acc, prop = e.get_mc_statistics()
                print(json.dumps(dict(K=K, N=512, sequence_move=m, round=r, iterations_per_s=a.iterations / dt,
                                      mix_ms_per_iteration=pt['mix_ms'] / a.iterations,
                                      propagate_ms_per_iteration=pt['propagate_ms'] / a.iterations,
                                      mc_acceptance=[float(acc[:, j].sum() / max(prop[:, j].sum(), 1)) for j in range(2)] if m else None,
                                      gpu=gpu, power_limit=power)), flush=True)
        for m, s in runs.items():
            print(json.dumps(dict(K=K, N=512, sequence_move=m, profiler=True, **kernel_ms(s, it[m], a.iterations), gpu=gpu,
                                  power_limit=power)), flush=True)
            it[m] += a.iterations


if __name__ == '__main__':
    main()
