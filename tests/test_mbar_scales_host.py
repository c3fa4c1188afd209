"""MBAR at the energy scales of real runs, without a GPU: the 50-digit mpmath MBAR of tests/mbar_mp.py against the
log-space oracle of oracle/mbar.py, and multistate.mbar.MBAR's solver with its two device passes replaced by that oracle.

The problems put states 10 to 10^4 kT apart, shift whole samples by up to 10^6 kT, model temperature ladders over 1000
and 4096 atoms, and place states without samples 900 kT beyond the ends."""
import numpy as np
import pytest

import mbar_mp as mm
from oracle import mbar as om
from openmmtools_b200.multistate.mbar import MBAR

EPS = np.finfo(np.float64).eps

# small enough for the mpmath reference (K <= 6, N <= 300), one per energy scale
SMALL = {
    'offsets_10': lambda: mm.offsets(4, 60, 10.0, 1),
    'offsets_40': lambda: mm.offsets(4, 60, 40.0, 2),
    'offsets_700': lambda: mm.offsets(4, 60, 700.0, 3),
    'offsets_1e4': lambda: mm.offsets(4, 60, 1.0e4, 4),
    'per_sample_1e5': lambda: mm.offsets(3, 80, 100.0, 5, d=-1.0e5, d_spread=100.0),
    'per_sample_1e6': lambda: mm.offsets(3, 80, 1000.0, 6, d=1.0e6, d_spread=1.0e6),
    'ladder_1000_atoms_unsampled_900': lambda: mm.temperature_ladder(1000, 300.0, 360.0, 4, 60, 7, unsampled=900.0),
}


class HostMBAR(MBAR):
    """multistate.mbar.MBAR with its device passes done by the log-space oracle, on u_kn shifted per sample by the
    lowest sampled energy as the device shifts it: the solver's own logic, at any scale, without a GPU."""

    def __init__(self, u_kn, N_k, initial_f_k=None, maximum_iterations=10000, relative_tolerance=1.0e-12):
        self.u_kn = np.asarray(u_kn, dtype=np.float64)
        self.N_k = np.asarray(N_k, dtype=np.int64)
        self._m = self.u_kn[self.N_k > 0].min(axis=0)
        self._u = self.u_kn - self._m[None, :]
        self._start(None, initial_f_k, maximum_iterations, relative_tolerance)

    def _evaluate(self, f, hessian):
        N, s = self.N_k.astype(np.float64), self.N_k > 0
        logD = om.log_denominator(self._u, self.N_k, f)
        lw = om.log_wsum(self._u, self.N_k, f)
        with np.errstate(over='ignore', invalid='ignore'):      # unsampled states far below: expm1 = inf, g = 0
            g = np.where(s, -N * np.expm1(lw), 0.0)
        H = None
        if hessian:
            W = np.exp(f[s, None] - self._u[s] - logD[None, :])
            H = np.zeros((len(f), len(f)))
            H[np.ix_(s, s)] = N[s, None] * N[None, s] * (W @ W.T) - np.diag(N[s] * np.exp(lw[s]))
        return float(np.sum(logD - self._m)), g, H, lw

    def _gram(self, f):
        W = om.weights(self._u, self.N_k, f)
        return W.T @ W, np.exp(om.log_wsum(self._u, self.N_k, f))


@pytest.fixture(scope='module')
def references():
    """{name: (u, N_k, mpmath Reference, its solution f as mpf)}, built once (about a second each)."""
    out = {}
    for name, make in SMALL.items():
        u, N_k = make()
        ref = mm.Reference(u, N_k)
        out[name] = (u, N_k, ref, ref.solve())
    return out


def _f64(f):
    return np.array([float(x) for x in f])


@pytest.mark.parametrize('name', list(SMALL))
def test_oracle_evaluation_matches_mpmath(references, name):
    u, N_k, ref, f_mp = references[name]
    us = om.shift_samples(u, N_k)
    for f in (np.zeros(len(N_k)), _f64(f_mp)):
        r = ref.evaluate(f)
        # log D_n: logsumexp of c_k - u_kn, each difference rounded at the size of its operands
        c = np.abs(np.log(np.maximum(N_k, 1)) + f)[:, None] + np.abs(u)
        scale = np.maximum(np.abs(r['logD']), c[N_k > 0].max(axis=0))
        assert np.all(np.abs(om.log_denominator(u, N_k, f) - r['logD']) <= 8 * EPS * scale)
        # on the shifted u the exp arguments are of the order of the spread across states, not of |u|: log sum W to
        # 1e-12 of max(1, |log sum W|), every state finite however far from f
        lw = om.log_wsum(us, N_k, f)
        assert np.all(np.isfinite(lw))
        assert np.all(np.abs(lw - r['log_wsum']) <= 1e-12 * np.maximum(1.0, np.abs(r['log_wsum'])))
        # G at the solution (sums of W up to 1): 1e-12 relative where it is a normal double
        if f is not None and np.array_equal(f, _f64(f_mp)):
            _, _, _, G, _, _ = om.evaluate(us, N_k, f)
            normal = np.abs(r['G']) >= np.finfo(np.float64).tiny
            assert np.all(np.abs(G - r['G'])[normal] <= 1e-12 * np.abs(r['G'])[normal])


@pytest.mark.parametrize('name', list(SMALL))
def test_oracle_solution_matches_mpmath(references, name):
    u, N_k, ref, f_mp = references[name]
    f_ref = _f64(f_mp)
    D, dD, f = om.free_energy_differences(u, N_k)
    # f carries the rounding of exp arguments of the order of the spread: 1e-12 of max(1, |f|)
    assert np.all(np.abs(f - f_ref) <= 1e-12 * np.maximum(1.0, np.abs(f_ref))), np.abs(f - f_ref).max()
    # dDelta_f: 1e-9 relative (the covariance goes through an eigendecomposition and an inverse of a K x K matrix);
    # pairs of states that are exact shifts of each other have dDelta_f = 0 up to rounding
    dd = ref.ddf(f_mp)
    big = dd > 1e-6 * dd.max()
    np.testing.assert_allclose(dD[big], dd[big], rtol=1e-9)
    assert np.all(dD[~big] <= 1e-6 * dd.max())


@pytest.mark.parametrize('name', list(SMALL))
def test_solver_matches_mpmath(references, name):
    u, N_k, ref, f_mp = references[name]
    f_ref = _f64(f_mp)
    m = HostMBAR(u, N_k)
    assert np.all(np.abs(m.f_k - f_ref) <= 1e-12 * np.maximum(1.0, np.abs(f_ref))), np.abs(m.f_k - f_ref).max()
    dd = ref.ddf(f_mp)
    big = dd > 1e-6 * dd.max()
    np.testing.assert_allclose(m.compute_free_energy_differences()['dDelta_f'][big], dd[big], rtol=1e-9)


# the rows of the scale table: every one is solved from f = 0 with the default relative_tolerance of 1e-12
TABLE = {
    'offsets_38': lambda: mm.offsets(4, 500, 38.0, 11),
    'offsets_40': lambda: mm.offsets(4, 500, 40.0, 12),
    'offsets_100': lambda: mm.offsets(4, 500, 100.0, 13),
    'offsets_700': lambda: mm.offsets(4, 500, 700.0, 14),
    'offsets_1e4': lambda: mm.offsets(4, 500, 1.0e4, 15),
    'ladder_1000_atoms_K8': lambda: mm.temperature_ladder(1000, 300.0, 360.0, 8, 500, 16),
    'ladder_1000_atoms_K64': lambda: mm.temperature_ladder(1000, 300.0, 360.0, 64, 500, 17),
    'ladder_4096_atoms_K64_unsampled_900': lambda: mm.temperature_ladder(4096, 300.0, 600.0, 64, 500, 18,
                                                                         unsampled=900.0),
    'per_sample_4e4': lambda: mm.offsets(4, 500, 10.0, 19, d=-4.0e4),
    'per_sample_1e5': lambda: mm.offsets(4, 500, 10.0, 20, d=-1.0e5, d_spread=100.0),
}


def check_solution(u, N_k, f, n_iterations):
    """f solves the MBAR equations as the log-space oracle evaluates them, and equals the oracle's own solution where
    its root finder, started from 20 self-consistent steps, reaches one (K <= 8: the 64-state ladders are too far off
    from there).  The residual |1 - sum_n W_in| is bounded by the solver's stopping rule, max(1e-12, 16 eps max|f|),
    plus the rounding of one more evaluation."""
    N_k = np.asarray(N_k)
    s = N_k > 0
    assert np.all(np.isfinite(f)) and f[0] == 0.0 and n_iterations < 200
    us = om.shift_samples(u, N_k)
    fg = f - f[s][0]
    bound = 2 * max(1e-12, 16 * EPS * np.abs(fg[s]).max())
    assert np.abs(np.expm1(om.log_wsum(us, N_k, fg)[s])).max() <= bound
    f0 = np.where(s, fg, 0.0)
    np.testing.assert_allclose(fg[~s], -om.log_wsum(us, N_k, f0)[~s], rtol=1e-12, atol=1e-12)
    if len(N_k) <= 8:
        f_o = om.solve(u, N_k)
        assert np.all(np.abs(f - f_o) <= 1e-11 * np.maximum(1.0, np.abs(f_o))), np.abs(f - f_o).max()


@pytest.mark.parametrize('name', list(TABLE))
def test_solver_at_the_scales_of_real_runs(name):
    u, N_k = TABLE[name]()
    m = HostMBAR(u, N_k)
    check_solution(u, N_k, m.f_k, m.n_iterations)
    if N_k[0] == 0:                 # the unsampled ends are exact shifts of their neighbours by 900 kT
        assert abs(m.f_k[1] - m.f_k[0] - 900.0) <= 1e-12 * abs(m.f_k[1])
        assert abs(m.f_k[-1] - m.f_k[-2] - 900.0) <= 1e-12 * abs(m.f_k[-1])


def test_two_state_pure_offset_gives_the_offset():
    """Row 1 = row 0 + Delta exactly (u on a grid of 2^-20 below 2^6, Delta an integer), so f_1 - f_0 = Delta."""
    rng = np.random.default_rng(3)
    for delta in (40.0, 700.0, 1.0e4):
        u0 = np.round(rng.normal(0.0, 1.0, 1000) * 2.0 ** 20) / 2.0 ** 20
        u = np.stack([u0, u0 + delta])
        m = HostMBAR(u, [500, 500])
        assert abs(m.f_k[1] - delta) <= 4 * EPS * delta
