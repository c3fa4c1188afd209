"""Monte Carlo rigid-body moves without a GPU: the proposal maps, the accept rule, signatures and state keys against the
reference (tests/golden/mc_moves_golden.npz, lifted by tests/golden/make_mc_moves_golden.py), the host restatement of
the device kernels (tests/mc_oracle.py) against the same, the SequenceMove shapes the engine runs, subset checks, and
storage of the moves with their statistics."""
import inspect
import json
import os
import numpy as np
import pytest
import mc_oracle as mo
from openmmtools_b200 import mcmc, unit
from openmmtools_b200.multistate import MultiStateReporter

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mc_moves_golden.npz'))
META = json.loads(str(G['meta']))


@pytest.fixture
def injected(monkeypatch):
    """np.random.randn / rand return the queued draws (the golden data's)."""
    queue = []
    monkeypatch.setattr(np.random, 'randn', lambda n: np.asarray(queue.pop(0))[:n])
    monkeypatch.setattr(np.random, 'rand', lambda n=None: np.asarray(queue.pop(0))[:n])
    return queue


def test_proposal_maps_match_reference(injected):
    P = unit.Quantity(G['positions'], unit.nanometer)
    for s, r, ref in zip(G['sigma'], G['randn'], G['displaced']):
        injected.append(r)
        out = mcmc.MCDisplacementMove.displace_positions(P, s * unit.nanometer)
        assert np.allclose(out / unit.nanometer, ref, rtol=0, atol=1e-15)
    for r, q, ref in zip(G['rand_q'], G['quaternions'], G['rotated']):
        injected.append(r)
        assert np.allclose(mcmc.MCRotationMove._generate_uniform_quaternion(), q, rtol=0, atol=1e-15)
        injected.append(r)
        assert np.allclose(mcmc.MCRotationMove.rotate_positions(P) / unit.nanometer, ref, rtol=0, atol=1e-14)
    for q, R in zip(G['q_cases'], G['matrices']):
        assert np.allclose(mcmc.MCRotationMove._rotation_matrix_from_quaternion(q), R, rtol=0, atol=1e-15)


def test_oracle_matches_reference():
    P = G['positions']
    for s, r, ref in zip(G['sigma'], G['randn'], G['displaced']):
        new, ok = mo.propose(mo.DISPLACEMENT, P, np.arange(len(P)), s * r, store=np.float64)
        assert ok and np.allclose(new, ref, rtol=0, atol=1e-15)
    for r, q, ref in zip(G['rand_q'], G['quaternions'], G['rotated']):
        assert np.allclose(mo.quaternion(r), q, rtol=0, atol=1e-15)
        new, ok = mo.propose(mo.ROTATION, P, np.arange(len(P)), mo.rotation_matrix(q), store=np.float64)
        assert ok and np.allclose(new, ref, rtol=0, atol=1e-14)
    for q, R in zip(G['q_cases'], G['matrices']):
        assert np.allclose(mo.rotation_matrix(q), R, rtol=0, atol=1e-15)
    for (e0, e1, u), (n_acc, n_prop, moved) in zip(G['accept_cases'], G['accepted']):
        assert mo.accept(e1 - e0, 1.0, u) == bool(n_acc) == bool(moved)


def test_oracle_rotation_makes_a_periodic_subset_whole():
    box = np.array([2.0, 2.0, 2.0])
    x = np.array([[0.05, 1.0, 1.0], [1.95, 1.0, 1.0], [0.1, 1.1, 1.0]])
    new, ok = mo.propose(mo.ROTATION, x, [0, 1, 2], mo.rotation_matrix([0.0, 0.0, 0.0, 1.0]), box, store=np.float64)
    assert ok     # a half turn about z of a subset that straddles the boundary: offsets -0.1 .. 0.05 from atom 0
    d = new[[1, 2]] - new[0]
    d -= box * np.round(d / box)
    assert np.allclose(np.linalg.norm(d, axis=1), [0.1, np.hypot(0.05, 0.1)])
    # offset (0.8, 0.8, 0) turned by 45 degrees about z: (0, 1.13, 0), past half the 1.9 nm edge
    far = np.array([[0.1, 0.1, 0.1], [0.9, 0.9, 0.1]])
    eighth = mo.rotation_matrix([np.cos(np.pi / 8), 0.0, 0.0, np.sin(np.pi / 8)])
    assert not mo.propose(mo.ROTATION, far, [0, 1], eighth, np.full(3, 1.9))[1]
    assert mo.propose(mo.ROTATION, far, [0, 1], eighth, np.full(3, 2.3))[1]


def test_signatures_and_state_keys_match_reference():
    for cls, sig in META['signatures'].items():
        params = [p for p in inspect.signature(getattr(mcmc, cls).__init__).parameters.values() if p.name != 'self']
        named = [[p.name, None if p.default is inspect.Parameter.empty else p.default] for p in params
                 if p.kind is not inspect.Parameter.VAR_KEYWORD]
        assert [n for n, _ in named] == [n for n, _ in sig['args']], cls
        for (n, d), (_, ref) in zip(named, sig['args']):
            if ref == 'None':
                assert d is None, (cls, n)
            elif ref is not None:
                assert np.isclose(unit.to_md(d), unit.to_md(eval(ref, {'unit': unit}))), (cls, n)
        assert (params[-1].kind is inspect.Parameter.VAR_KEYWORD) == (sig['kwarg'] is not None), cls
    moves = dict(MetropolizedMove=mcmc.MetropolizedMove(), MCDisplacementMove=mcmc.MCDisplacementMove(),
                 MCRotationMove=mcmc.MCRotationMove(), SequenceMove=mcmc.SequenceMove([mcmc.MCRotationMove()]))
    for cls, keys in META['state_keys'].items():
        assert sorted(moves[cls].__getstate__()) == keys, cls


def lang(n=10):
    return mcmc.LangevinSplittingDynamicsMove(n_steps=n)


def test_sequence_shapes():
    d, r = mcmc.MCDisplacementMove(atom_subset=[0]), mcmc.MCRotationMove(atom_subset=[0, 1])
    dyn = lang()
    assert mcmc.split_move(mcmc.SequenceMove([d, r, dyn])) == ([d, r], dyn)
    mc, integrator = mcmc.split_move(mcmc.SequenceMove([d, r]))
    assert mc == [d, r] and integrator is None
    assert mcmc.integrator_part(mcmc.SequenceMove([d])).n_steps == 0
    assert mcmc.split_move(d) == ([d], None)
    assert mcmc.split_move(mcmc.SequenceMove([lang()]))[0] == []
    assert len(mcmc.split_move(mcmc.SequenceMove([d] * 4 + [lang()]))[0]) == 4
    for bad, why in (([lang(), d], 'after the dynamics'), ([lang(), lang()], 'two integrator moves'),
                     ([d] * 5, '5 Monte Carlo moves'), ([mcmc.SequenceMove([d])], 'inside a SequenceMove')):
        with pytest.raises(NotImplementedError, match=why):
            mcmc.split_move(mcmc.SequenceMove(bad))
    s = mcmc.SequenceMove([d, r, lang()])
    assert list(s) == s.move_list and str(s) == str(s.move_list)
    assert s.statistics == [dict(n_accepted=0, n_proposed=0)] * 2 + [{}]
    s.statistics = [dict(n_accepted=1, n_proposed=2), dict(n_accepted=3, n_proposed=4), {}]
    assert (d.n_accepted, d.n_proposed, r.n_accepted, r.n_proposed) == (1, 2, 3, 4)


def test_subset_checks():
    assert np.array_equal(mcmc.MCRotationMove().subset_indices(4), np.arange(4))
    assert np.array_equal(mcmc.MCRotationMove(atom_subset=slice(1, 3)).subset_indices(4), [1, 2])
    assert np.array_equal(mcmc.MCRotationMove(atom_subset=[3]).subset_indices(4), [3])
    for bad in ([4], [-1], [1, 1], [], slice(5, 9), [0.5]):
        with pytest.raises(ValueError):
            mcmc.MCRotationMove(atom_subset=bad).subset_indices(4)
    for sigma in (-0.1, np.inf, np.nan):
        with pytest.raises(ValueError):
            mcmc.MCDisplacementMove(displacement_sigma=sigma * unit.nanometer)._engine_move(4)
    kind, sigma, idx = mcmc.MCDisplacementMove(displacement_sigma=2.0 * unit.angstrom, atom_subset=[2])._engine_move(4)
    assert kind == mo.DISPLACEMENT and np.isclose(sigma, 0.2) and list(idx) == [2]


def test_sequence_with_statistics_round_trips_through_storage(tmp_path):
    s = mcmc.SequenceMove([mcmc.MCDisplacementMove(displacement_sigma=0.3 * unit.nanometer, atom_subset=slice(0, 4)),
                           mcmc.MCRotationMove(atom_subset=[0, 1, 2, 3]), lang(500)])
    s.statistics = [dict(n_accepted=7, n_proposed=20), dict(n_accepted=2, n_proposed=20), {}]
    r = MultiStateReporter(str(tmp_path / 'run'), open_mode='w')
    r.write_mcmc_moves([s, s])
    back = MultiStateReporter(str(tmp_path / 'run'), open_mode='r').read_mcmc_moves()
    assert len(back) == 2 and back[0].statistics == s.statistics
    d = back[0].move_list[0]
    assert d.atom_subset == slice(0, 4) and np.isclose(unit.to_md(d.displacement_sigma), 0.3)
    assert back[0].move_list[2].n_steps == 500
