"""Decouple toluene from OBC implicit solvent: iterations/s, per-phase times and the free energy of decoupling.

For TolueneImplicit (OBC1) and TolueneImplicitOBC2, the whole molecule alchemical, a ladder of M states (first
lambda_electrostatics 1 -> 0, then lambda_sterics 1 -> 0) sampled by ReplicaExchangeSampler with K = M replicas,
LangevinSplittingDynamicsMove (2 fs, 500 steps, HBonds constraints), swap-all mixing.  After `--warmup` iterations,
`--iterations` are timed with a host clock around sampler.run (which ends in a device synchronise), the phase split from the
engine's CUDA events.  The stored run is then analysed by ReplicaExchangeAnalyzer: Delta f (decoupled - coupled) +- its
error, in kT.  Prints one JSON line per (system, M), with the card's name and power limit.
Usage: python tools/run_alchemical_molecule.py [--states 64,128] [--iterations 200] [--warmup 20] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmmtools_b200 import alchemy, mcmc, multistate, states, testsystems, unit  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the timing itself needs no nvidia-smi
        return 'unknown (%s)' % e


def ladder(M):
    ne = M // 2
    le = list(np.linspace(1.0, 0.0, ne)) + [0.0] * (M - ne)
    ls = [1.0] * ne + list(np.linspace(1.0, 0.0, M - ne + 1)[1:])
    return {'lambda_electrostatics': le, 'lambda_sterics': ls}


def run(name, cls, M, n_iter, warmup, path):
    t = cls()
    asys = alchemy.AbsoluteAlchemicalFactory().create_alchemical_system(
        t.system, alchemy.AlchemicalRegion(alchemical_atoms=range(t.system.n_particles)))
    tss = states.create_thermodynamic_state_protocol(asys, ladder(M), constants={'temperature': 300 * unit.kelvin},
                                                     composable_states=alchemy.AlchemicalState.from_system(asys))
    move = mcmc.LangevinSplittingDynamicsMove(timestep=2.0 * unit.femtosecond, n_steps=500)
    s = multistate.ReplicaExchangeSampler(mcmc_moves=move, number_of_iterations=warmup + n_iter, seed=7)
    s.create(tss, [states.SamplerState(t.positions)], storage=multistate.MultiStateReporter(path, checkpoint_interval=50))
    s.minimize(max_iterations=200)
    s.run(warmup)
    s._engine.phase_times(reset=True)
    t0 = time.perf_counter()
    s.run(n_iter)
    wall = time.perf_counter() - t0
    ph = s._engine.phase_times()
    del s
    a = multistate.ReplicaExchangeAnalyzer(multistate.MultiStateReporter(path, open_mode='r'))
    D, dD = a.get_free_energy()
    per = lambda k: ph[k] / n_iter
    return dict(system=name, states=M, replicas=M, atoms=asys.n_particles, iterations=n_iter,
                iterations_per_s=n_iter / wall, ms_per_iteration=1e3 * wall / n_iter,
                mix_ms=per('mix_ms'), propagate_ms=per('propagate_ms'), energies_ms=per('energies_ms'),
                energies_share_of_iteration=per('energies_ms') / (1e3 * wall / n_iter),
                delta_f_kT=float(D[0, -1]), d_delta_f_kT=float(dD[0, -1]), card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--states', default='64,128')
    ap.add_argument('--iterations', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--out', default=None, help='directory for the runs (default: a temporary one)')
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp()
    for name, cls in (('TolueneImplicit (OBC1)', testsystems.TolueneImplicit), ('TolueneImplicitOBC2', testsystems.TolueneImplicitOBC2)):
        for M in (int(v) for v in args.states.split(',')):
            path = os.path.join(out, '%s-%d.nc' % (name.split()[0], M))
            print(json.dumps(run(name, cls, M, args.iterations, args.warmup, path)), flush=True)


if __name__ == '__main__':
    main()
