"""Cost of hybrid Monte Carlo against Langevin dynamics at the same number of velocity-Verlet / Langevin steps on two
shapes: the headline 512-atom alchemical LJ fluid (5 alchemical atoms) at K = 256 replicas, swap-all, and config 4's
AlanineDipeptideVacuum (HBonds) parallel tempering at K = 128, 300-600 K.  HMCMove(n_steps=n) takes n trials of n
velocity-Verlet steps per iteration: n^2 force evaluations, plus one at the first trial and after each rejection (on a
molecule also two f64 energy passes per trial); the Langevin move runs n^2 steps of "V R O R V" at the same timestep.

Prints one JSON line per (workload, move, timestep, round): ms per iteration of the fused device loop (rx_run_iterations),
steps per iteration, and for HMC the acceptance rate of the trials of the timed iterations, with the card's name and
power limit.
usage: run_hmc.py [--workloads lj config4] [--K 256] [--K4 128] [--n 20] [--iterations 10] [--rounds 2] [--timesteps 1 2]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openmmtools_b200 import testsystems, alchemy, states, mcmc, multistate, unit


def sampler(K, move):
    fluid = testsystems.LennardJonesFluid(nparticles=512)
    asys = alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=True).create_alchemical_system(
        fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(5)))
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': [1.0 - l / (K - 1) for l in range(K)]}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=alchemy.AlchemicalState.from_system(asys))
    sstate = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=10 ** 9, replica_mixing_scheme='swap-all', seed=1234)
    s.create(tstates, [sstate], storage=None)
    s.minimize(max_iterations=200)
    s._compute_energies()
    return s


def sampler_config4(K, move):
    a = testsystems.AlanineDipeptideVacuum()
    ts = states.ThermodynamicState(a.system, 300.0 * unit.kelvin)
    s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=10 ** 9, seed=1234)
    s.create(ts, [states.SamplerState(a.positions)], storage=None, min_temperature=300.0 * unit.kelvin,
             max_temperature=600.0 * unit.kelvin, n_temperatures=K)
    s._compute_energies()
    return s


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [t.strip() for t in out.split(',')]
        return name, power
    except Exception as e:   # (the numbers below are still device times)
        return 'unknown (%s)' % e, 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', nargs='+', default=['lj', 'config4'], choices=['lj', 'config4'])
    ap.add_argument('--K', type=int, default=256)
    ap.add_argument('--K4', type=int, default=128)
    ap.add_argument('--n', type=int, default=20)
    ap.add_argument('--iterations', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--timesteps', type=float, nargs='+', default=[1.0, 2.0])
    a = ap.parse_args()
    name, power = card()
    runs = []
    for wl in a.workloads:
        make, K, atoms, gamma = (sampler, a.K, 512, 10.0) if wl == 'lj' else (sampler_config4, a.K4, 22, 5.0)
        for fs in a.timesteps:
            runs.append((wl, K, atoms, 'hmc', fs, make(K, mcmc.HMCMove(timestep=fs * unit.femtosecond, n_steps=a.n))))
            runs.append((wl, K, atoms, 'langevin', fs, make(K, mcmc.LangevinSplittingDynamicsMove(
                timestep=fs * unit.femtosecond, collision_rate=gamma / unit.picosecond, n_steps=a.n * a.n))))
    first = {id(r[-1]): 1 for r in runs}
    for *_, s in runs:   # warm-up: every shape once
        s._engine.run_iterations(1, 'swap-all', s._seed, 1)
        first[id(s)] = 2
    for rnd in range(a.rounds):
        for wl, K, atoms, kind, fs, s in runs:   # alternated in one process
            e = s._engine
            acc0, n0 = e.get_hmc_statistics() if kind == 'hmc' else (None, None)
            t = time.perf_counter()
            e.run_iterations(a.iterations, 'swap-all', s._seed, first[id(s)])
            e.get_replica_states()   # (ends in a device synchronise)
            ms = (time.perf_counter() - t) * 1e3 / a.iterations
            first[id(s)] += a.iterations
            rec = dict(workload=wl, move=kind, timestep_fs=fs, K=K, atoms=atoms, steps_per_iteration=a.n * a.n, round=rnd,
                       ms_per_iteration=round(ms, 3), card=name, power_limit=power)
            if kind == 'hmc':
                acc1, n1 = e.get_hmc_statistics()
                rec.update(n_steps=a.n, trials=int((n1 - n0).sum()), acceptance=round(float((acc1 - acc0).sum() / (n1 - n0).sum()), 4))
            print(json.dumps(rec), flush=True)


if __name__ == '__main__':
    main()
