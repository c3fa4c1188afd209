"""Small end-to-end workload for compute-sanitizer (memcheck / racecheck / initcheck): every kernel runs at least once."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden'))
import numpy as np
from energy_models import energies
from openmmtools_b200 import testsystems, alchemy, states, mcmc, multistate, unit
from openmmtools_b200._engine import Engine

# mixing kernels: pow2 small, K=256 (row image, k_mix_walk2 + k_mix_walk_pow2<true> tail), K not a power of two (k_cand_* + k_mix_walk2c + plain tail;
# above 256 k_cand_records<true> + k_mix_walk_cand), neighbours
for K, n in ((16, 4096), (256, 60000), (12, 1728), (100, 30000), (255, 20000), (300, 20000)):
    e = Engine(0, K, K)
    e.set_energies(energies('flat', K, 7)); e.set_replica_states(np.arange(K)); e.mix_seed(3, 0); e.mix_seed(4, 1)
    e.mix_swap_all(n); e.mix_swap_all(n); e.mix_swap_neighbors()
    e.selftest_exp(np.linspace(-40.0, 0.0, 64))
    e.close()
# sampler: LJ alchemical (propagate with Verlet list, energies) and harmonic oscillator
fluid = testsystems.LennardJonesFluid(nparticles=128)
asys = alchemy.AbsoluteAlchemicalFactory().create_alchemical_system(fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(4)))
K = 8
ts = states.create_thermodynamic_state_protocol(asys, {'lambda_sterics': [1 - l / (K - 1) for l in range(K)]},
                                                constants={'temperature': 300 * unit.kelvin},
                                                composable_states=alchemy.AlchemicalState.from_system(asys))
ss = states.SamplerState(fluid.positions, box_vectors=asys.getDefaultPeriodicBoxVectors())
s = multistate.ReplicaExchangeSampler(mcmc_moves=mcmc.LangevinSplittingDynamicsMove(n_steps=12), number_of_iterations=3, seed=1)
s.create(ts, [ss]); s.run(); s.sampler_states
s._engine.run_iterations(2, 'swap-all', 1, 10)
s._engine.set_integrator(0.002, 1.0, 150, 'V R O R V')  # long enough for list re-partitions and an outer rebuild
s._engine.run_iterations(1, 'swap-all', 1, 12)
# one move per state (k_propagate<.., PS>), the NaN restart path
s._engine.set_state_integrator(3, 0.001, 5.0, 20, 'O V R V O', True)
s._engine.run_iterations(1, 'swap-all', 1, 13)
s._engine.set_integrator(0.002, 1.0, 12, 'V R O R V')
s._engine.propagate(1, 14); s._engine.propagate_retry(2, 14)
ho = testsystems.HarmonicOscillator()
hs = multistate.ReplicaExchangeSampler(mcmc_moves=mcmc.LangevinSplittingDynamicsMove(n_steps=20), number_of_iterations=2, seed=2,
                                       replica_mixing_scheme='swap-neighbors')
hs.create([states.ThermodynamicState(ho.system, T * unit.kelvin) for T in (300, 310, 320)], [states.SamplerState(ho.positions)])
hs.run()
# SAMS on the device (k_sams_step): 2 replicas over 3 oscillator states, per-iteration and fused
ss_ = multistate.SAMSSampler(mcmc_moves=mcmc.LangevinSplittingDynamicsMove(n_steps=20), number_of_iterations=10 ** 6, seed=5,
                             flatness_criteria='minimum-visits', device_weight_update=True)
ss_.create([states.ThermodynamicState(ho.system, T * unit.kelvin) for T in (300, 310, 320)], [states.SamplerState(ho.positions)] * 2)
ss_.run(6); ss_.run_fused(4)
# energy history and the u_kn gather (k_mbar_gather): partial tiles in both directions, two unsampled columns
from openmmtools_b200.multistate.mbar import MBAR
e = Engine(0, 7, 40)
rng = np.random.default_rng(0)
e.history_load(rng.normal(size=(50, 7, 40)), rng.normal(size=(50, 7, 2)))
N_k = np.zeros(42, np.int64); N_k[1:8] = 37
MBAR.from_history(e, np.arange(3, 40), np.r_[40, np.arange(40), 41], N_k).close()
# the per-sample shift (k_mbar_shift) and the log-space row sums over several chunks (k_mbar_rowsum, k_mbar_tree_rows)
# on a host-built u_kn with a partial last chunk, states 800 kT apart and unsampled ends
u = rng.normal(size=(5, 3 * 8192 + 5)) + np.array([-900.0, 0.0, 400.0, 800.0, 1700.0])[:, None] - 1.0e5
MBAR(u, [0, 8192, 8192, 8197, 0]).close()
e.close()
# alchemical molecules (ALCH instantiations): OBC2 with a partial region, vacuum with the whole molecule -- Langevin,
# HMC, Monte Carlo moves, FIRE, energy rows at sampled and unsampled states
for cls, atoms in ((testsystems.TolueneImplicitOBC2, [0, 3, 9, 10]), (testsystems.TolueneVacuum, range(15))):
    tol = cls()
    amol = alchemy.AbsoluteAlchemicalFactory().create_alchemical_system(tol.system, alchemy.AlchemicalRegion(alchemical_atoms=atoms))
    ats = states.create_thermodynamic_state_protocol(amol, {'lambda_electrostatics': [1.0, 0.5, 0.0, 0.0], 'lambda_sterics': [1.0, 1.0, 0.5, 0.0]},
                                                     constants={'temperature': 300 * unit.kelvin},
                                                     composable_states=alchemy.AlchemicalState.from_system(amol))
    for mv in (mcmc.LangevinSplittingDynamicsMove(n_steps=10), mcmc.HMCMove(n_steps=3),
               mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.01 * unit.nanometer, atom_subset=list(range(15))),
                                  mcmc.MCRotationMove(atom_subset=list(range(15)))])):
        ms = multistate.ReplicaExchangeSampler(mcmc_moves=mv, number_of_iterations=2, seed=3)
        ms.create(ats, [states.SamplerState(tol.positions)], unsampled_thermodynamic_states=[ats[0], ats[-1]])
        ms.minimize(max_iterations=20); ms.run()
print('sanitize workload done')
