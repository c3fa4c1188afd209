"""BASELINE.json configs[3]: T-REMD of testsystems.AlanineDipeptideVacuum, 128 temperature replicas 300-600 K, 1000 steps per
iteration (ParallelTemperingSampler, swap-all), timed on one GPU; energies of the final configurations checked against the
oracle.  usage: run_config4.py [--implicit] [iterations [K [n_steps]]]
--implicit: AlanineDipeptideImplicit (OBC1 implicit solvent) in place of the vacuum system.  The card's name and power limit
are printed with the times."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import zlib
import numpy as np
rank, world = int(os.environ.get('RANK', '0')), int(os.environ.get('WORLD_SIZE', '1'))
if world > 1:
    import torch, torch.distributed as dist
    torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
    dist.init_process_group('nccl')
if rank != 0:
    sys.stdout = open(os.devnull, 'w')
from openmmtools_b200 import testsystems, states, mcmc, multistate, unit
from oracle import oracle, implicit as oracle_implicit

implicit = '--implicit' in sys.argv
sys.argv = [v for v in sys.argv if v != '--implicit']
n_it = int(sys.argv[1]) if len(sys.argv) > 1 else 10
K = int(sys.argv[2]) if len(sys.argv) > 2 else 128
n_steps = int(sys.argv[3]) if len(sys.argv) > 3 else 1000
KB = 8.31446261815324e-3
a = testsystems.AlanineDipeptideImplicit() if implicit else testsystems.AlanineDipeptideVacuum()
try:
    import subprocess
    print('card:', subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                                  text=True).stdout.strip().splitlines()[0], '| system:', type(a).__name__)
except (OSError, IndexError):
    print('card: unknown | system:', type(a).__name__)
ts = states.ThermodynamicState(a.system, 300.0 * unit.kelvin)
move = mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtosecond, collision_rate=5.0 / unit.picosecond, n_steps=n_steps)
s = multistate.ParallelTemperingSampler(mcmc_moves=move, number_of_iterations=10 ** 9, seed=7)
s.create(ts, [states.SamplerState(a.positions)], storage=None, min_temperature=300.0 * unit.kelvin,
         max_temperature=600.0 * unit.kelvin, n_temperatures=K)
s.run(3)
e = s._engine
e.phase_times(reset=True)
t0 = time.time(); s.run(n_it); dt = time.time() - t0
pt = e.phase_times()
print('%d GPU(s)  digest after %d iterations: replica states %08x  energy matrix %08x' % (
    world, s._iteration, zlib.crc32(np.ascontiguousarray(s._replica_thermodynamic_states, np.int64).tobytes()),
    zlib.crc32(np.ascontiguousarray(s._energy_thermodynamic_states, np.float64).tobytes())))
print('config 4: K=%d, %d steps/iteration: %.2f ms per iteration (%.1f iterations/s); device phases per iteration: mix %.3f propagate %.3f '
      'energies %.3f ms' % (K, n_steps, 1e3 * dt / n_it, n_it / dt, pt['mix_ms'] / n_it, pt['propagate_ms'] / n_it, pt['energies_ms'] / n_it))
e.phase_times(reset=True)
t0 = time.time(); e.run_iterations(n_it, 'swap-all', s._seed, s._iteration + 1); dt = time.time() - t0
print('fused device loop: %.2f ms per iteration (%.1f iterations/s)' % (1e3 * dt / n_it, n_it / dt))
m = (oracle_implicit if implicit else oracle).Molecule(a.system)
T = np.array([st.temperature.value_in_unit(unit.kelvin) for st in s._thermodynamic_states])
s._states_stale = True
u = e.compute_energies()
x = e.get_positions()       # (this rank's replicas)
err = max(np.abs(u[e.k0 + k] - m.energy(np.ascontiguousarray(x[k])) / (KB * T)).max() for k in range(len(x)))
c = a.system.constraints
i, j = c[:, 0].astype(int), c[:, 1].astype(int)
print('max |u - oracle| %.2e   max constraint error %.2e nm   acceptance %.3f' % (
    err, np.abs(np.linalg.norm(x[:, i] - x[:, j], axis=2) - c[None, :, 2]).max(),
    s._n_accepted_matrix.sum() / max(s._n_proposed_matrix.sum(), 1)))
t0 = time.time()
xo = np.ascontiguousarray(x[0]); vo = np.zeros_like(xo)
m.langevin(xo, vo, np.random.default_rng(0).normal(size=(n_steps, 22, 3)), KB * 300, 0.002, 5.0, n_steps, 'VRORV', tol=1e-8)
print('oracle (one host core): %.2f ms per replica-iteration -> %.1f ms per iteration for %d replicas on one core' % (
    1e3 * (time.time() - t0), 1e3 * (time.time() - t0) * K, K))
