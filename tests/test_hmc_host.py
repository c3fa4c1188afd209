"""Hybrid Monte Carlo without a GPU: the reference's HMCIntegrator program (tests/golden/make_hmc_golden.py, recorded from
the unmodified integrators.py) interpreted again, the host oracle trial against it, HMCMove's signature and serialisation,
split_move and the refusals, and the numpy regeneration of the device's HMC Philox streams."""
import json
import os
import sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
import hmc_oracle as ho
from helpers import KB, philox4x32_10, philox_normal3
from make_hmc_golden import CASES, case_inputs, interpret, program_from_text
from openmmtools_b200 import mcmc, unit

G = np.load(os.path.join(HERE, 'golden', 'hmc_golden.npz'))


def test_reference_program_is_the_documented_one():
    for idx, (_, nsteps, _, _, _) in enumerate(CASES):
        prog = [str(p) for p in G['case%d_program' % idx]]
        assert prog.count('perdof|v|v+0.5*dt*f/m') == nsteps and prog.count('perdof|x|x+dt*v') == nsteps
        assert prog.count('perdof|v|v+0.5*dt*f/m+(x-x1)/dt') == nsteps
        assert prog.index('update_context') < prog.index('perdof|v|sigma*gaussian')   # (a CM remover has no effect)
        assert 'global|accept|step(exp(-(Enew-Eold)/kT) - uniform)' in prog
        assert 'perdof|x|x*accept + xold*(1-accept)' in prog
        assert prog[-2:] == ['global|naccept|naccept + accept', 'global|ntrials|ntrials + 1']


@pytest.mark.parametrize('idx', range(len(CASES)))
def test_golden_program_reproduces(idx):
    nsteps = CASES[idx][1]
    x, mass, ef, gauss, unif, cons = case_inputs(idx)
    g0 = dict(zip([str(n) for n in G['case%d_global_names' % idx]], G['case%d_global_values' % idx]))
    res, g = interpret(program_from_text(G['case%d_program' % idx]), g0, float(G['case%d_dt' % idx]), x, mass, ef, gauss,
                       unif, nsteps, cons)
    assert np.array_equal(np.stack([r[0] for r in res]), G['case%d_x' % idx])
    assert np.array_equal(np.stack([r[1] for r in res]), G['case%d_v' % idx])
    assert np.array_equal(np.array([[r[2], r[3], r[4]] for r in res]), G['case%d_E' % idx])
    assert [g['naccept'], g['ntrials']] == list(G['case%d_counts' % idx])


@pytest.mark.parametrize('idx', range(len(CASES)))
def test_oracle_trial_matches_the_interpreted_reference_program(idx):
    kind, nsteps, dt, T, _ = CASES[idx]
    x, mass, ef, gauss, unif, cons = case_inputs(idx)
    kT = KB * T
    g0 = dict(zip([str(n) for n in G['case%d_global_names' % idx]], G['case%d_global_values' % idx]))
    assert abs(g0['kT'] - kT) < 1e-12 * kT
    for t in range(nsteps):
        x, v, e0, e1, acc = ho.trial(x, mass, kT, ef, gauss[t], unif[t], dt, nsteps, cons)
        assert np.abs(x - G['case%d_x' % idx][t]).max() < 1e-12
        assert np.abs(v - G['case%d_v' % idx][t]).max() < 1e-12
        if cons is not None and acc:   # the constraints hold (a rejection restores the start, which need not hold them)
            i, j = cons[:, 0].astype(int), cons[:, 1].astype(int)
            assert np.abs(np.linalg.norm(x[i] - x[j], axis=1) - cons[:, 2]).max() < 1e-10
            assert np.abs(np.einsum('cq,cq->c', x[i] - x[j], v[i] - v[j])).max() < 1e-8
        e_ref = G['case%d_E' % idx][t]
        assert abs(e0 - e_ref[0]) < 1e-12 * max(1.0, abs(e_ref[0])) and abs(e1 - e_ref[1]) < 1e-12 * max(1.0, abs(e_ref[1]))
        assert acc == bool(e_ref[2])


def test_golden_covers_the_constrained_molecule():
    kinds = [c[0] for c in CASES]
    assert 'aladip' in kinds
    prog = [str(p) for p in G['case%d_program' % kinds.index('aladip')]]
    assert prog.count('constrain_x') == CASES[kinds.index('aladip')][1] and 'constrain_v' in prog


def test_golden_has_rejected_and_accepted_trials():
    acc = np.concatenate([G['case%d_E' % i][:, 2] for i in range(len(CASES))])
    assert acc.min() == 0.0 and acc.max() == 1.0


def test_rejected_trial_keeps_nan_positions():
    """x*accept + xold*(1-accept) with accept = 0: xold where x is finite, NaN where it is not."""
    x = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]])

    def ef(y):
        d = y[1] - y[0]
        if np.linalg.norm(d) < 0.5:
            return np.nan, np.full_like(y, np.nan)
        return 0.0, np.zeros_like(y)
    xn, _, _, e1, acc = ho.trial(x, np.ones(2), 2.5, ef, np.array([[0.0, 0.0, 0.0], [-60.0, 0.0, 0.0]]), 0.5, 0.01, 2)
    assert not acc and np.isnan(e1) and np.isnan(xn).any()


def test_hmc_philox_streams_regenerate():
    seed, it = 0x1234_5678_9ABC, 7
    g, u = ho.draws(seed, it, 5, 16, 3)
    assert g.shape == (3, 16, 3) and u.shape == (3,)
    assert np.all((u > 0) & (u < 1)) and abs(g.mean()) < 0.5
    key = (seed & 0xFFFFFFFF, ((seed >> 32) ^ (it >> 32)) & 0xFFFFFFFF)
    one = philox_normal3(philox4x32_10(np.array([[7, 0x90000002, 5, it]], np.uint32), key))
    assert np.array_equal(one[0], g[2, 7])
    w = philox4x32_10(np.array([[1, 0xB0000000, 5, it]], np.uint32), key)
    assert u[1] == (float(w[0, 0]) + 0.5) * 2.0 ** -32
    # streams of other replicas, iterations and tags differ
    assert not np.array_equal(ho.draws(seed, it, 6, 16, 3)[0], g)
    assert not np.array_equal(ho.draws(seed, it + 1, 5, 16, 3)[1], u)


def test_hmc_move_signature_matches_the_reference():
    gold = json.load(open(os.path.join(HERE, 'golden', 'hmc_signatures_golden.json')))
    import inspect
    sig = inspect.signature(mcmc.HMCMove.__init__)
    args = [n for n, p in sig.parameters.items() if n != 'self' and p.kind == p.POSITIONAL_OR_KEYWORD]
    assert args == [a[0] for a in gold['mcmc.py:HMCMove.__init__']['args']]
    assert [a[1] for a in gold['mcmc.py:HMCMove.__init__']['args']] == ['1.0 * unit.femtosecond', '1000']
    assert gold['mcmc.py:HMCMove.__init__']['kwarg'] == 'kwargs'
    assert any(p.kind == p.VAR_KEYWORD for p in sig.parameters.values())
    m = mcmc.HMCMove()
    assert m.n_steps == 1000 and abs(unit.to_md(m.timestep, unit.picosecond) - 0.001) < 1e-15


def test_hmc_move_state_round_trip():
    m = mcmc.HMCMove(timestep=0.5 * unit.femtosecond, n_steps=10, n_restart_attempts=2)
    s = m.__getstate__()
    assert set(s) == {'n_steps', 'reassign_velocities', 'n_restart_attempts', 'timestep'}
    gold = json.load(open(os.path.join(HERE, 'golden', 'hmc_signatures_golden.json')))
    assert set(gold['mcmc.py:HMCMove.__getstate__']['keys']) <= set(s)
    m2 = mcmc.HMCMove.__new__(mcmc.HMCMove)
    m2.__setstate__(s)
    assert m2._integrator_parameters() == m._integrator_parameters() == (0.0005, 0.0, 10, 'HMC')


def test_split_move_takes_hmc():
    h = mcmc.HMCMove(n_steps=5)
    assert mcmc.split_move(h) == ([], h)
    d, r = mcmc.MCDisplacementMove(), mcmc.MCRotationMove()
    mc, integ = mcmc.split_move(mcmc.SequenceMove([d, r, h]))
    assert mc == [d, r] and integ is h
    mc, integ = mcmc.split_move(mcmc.SequenceMove([mcmc.MCDisplacementMove() for _ in range(4)] + [h]))
    assert len(mc) == 4 and integ is h
    with pytest.raises(NotImplementedError):
        mcmc.split_move(mcmc.SequenceMove([mcmc.MCDisplacementMove() for _ in range(5)] + [h]))
    with pytest.raises(NotImplementedError):
        mcmc.split_move(mcmc.SequenceMove([h, d]))
    with pytest.raises(NotImplementedError):
        mcmc.split_move(mcmc.SequenceMove([h, mcmc.LangevinDynamicsMove()]))


def test_hmc_refusals():
    h1, h2 = mcmc.HMCMove(timestep=1.0 * unit.femtosecond), mcmc.HMCMove(timestep=2.0 * unit.femtosecond)
    mcmc.check_hmc([h1, h2])                               # per-state timesteps
    mcmc.check_hmc([mcmc.LangevinDynamicsMove()], 1.0)     # (no HMC: nothing to refuse)
    with pytest.raises(NotImplementedError, match='mix'):
        mcmc.check_hmc([h1, mcmc.LangevinDynamicsMove()])
    with pytest.raises(NotImplementedError, match='mix'):
        mcmc.check_hmc([h1, mcmc.integrator_part(mcmc.MCDisplacementMove())])
    with pytest.raises(NotImplementedError, match='constant pressure'):
        mcmc.check_hmc([h1], pressure=1.0 * unit.atmosphere)
