"""MBAR free energies (Shirts & Chodera 2008) with both passes of every iteration on the GPU (rx_mbar_*, DESIGN §4.7).

For K states with N_k samples each, and u_kn the reduced potential of sample n in state k, the MBAR estimates f_k solve

    f_i = -log sum_n exp(-u_in) / D_n,    D_n = sum_k N_k exp(f_k - u_kn),

equivalently they maximise the concave log-likelihood  L(f) = sum_k N_k f_k - sum_n log D_n,  whose gradient
g_i = N_i - N_i sum_n W_in and Hessian H_ij = N_i N_j sum_n W_in W_jn - delta_ij N_i sum_n W_in use the weights
W_in = exp(f_i - u_in) / D_n.  The device evaluates log D_n, log sum_n W_in, g and H; the host takes self-consistent
steps (f_i <- f_i - log sum_n W_in) until the relative gradient is small, then Newton steps (a K x K solve in numpy), and
stops when max_i |g_i| / N_i = max_i |expm1(log sum_n W_in)| <= relative_tolerance, or <= 16 eps max_i |f_i|, the
rounding floor of that residual, where this is larger (f spread over more than ~300 kT).  A Newton step that the
Hessian cannot give or that no backtracking makes ascend is replaced by a self-consistent step.  The gauge is f_0 = 0.  The sums of
W are taken in log space and every sample is shifted by its lowest sampled energy on the device, so states tens to
thousands of kT apart and energies of |u| ~ 1e5 kT solve as well as energies of order 1 kT.

States without samples (N_k = 0) take no part in D_n; their f_k follow from the converged f of the others by the
equation above, from the log sums at f_k = 0.  The asymptotic covariance of f comes from the weight matrix W (N x K) through its SVD W = U S V^T,
with V and S from the eigendecomposition of the device Gram matrix W^T W = V S^2 V^T:

    Theta = W^T (I - W diag(N) W^T)^+ W = V S (I - S V^T diag(N) V S)^+ S V^T,
    dDelta_f_ij = sqrt(Theta_ii + Theta_jj - 2 Theta_ij).

(Subtracting W^T W = V S^2 V^T from Theta, as one variant of this formula does, makes dDelta_f of harmonic oscillators
about 2.3 times smaller than the spread of Delta_f over independent runs; tests/test_mbar_host.py checks the spread.)
"""
import ctypes as C

import numpy as np

from .. import _lib


class MBARConvergenceError(RuntimeError):
    """The MBAR equations were not solved to the requested tolerance."""


def _check(lib, h, rc):
    if rc != _lib.RX_OK:
        msg = lib.rx_mbar_last_error(h).decode()
        if rc == _lib.RX_ERR_UNSUPPORTED:
            raise NotImplementedError(msg)
        if rc == _lib.RX_ERR_INVALID:
            raise ValueError(msg)
        raise RuntimeError(msg)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class MBAR:
    """Multistate Bennett acceptance ratio estimator on the GPU.

    Parameters
    ----------
    u_kn : array (K, N) of reduced potentials (kT) of every sample in every state
    N_k : array (K,) of the samples drawn from each state, in the order of the columns of u_kn (zeros allowed)
    initial_f_k : array (K,), optional, starting guess (shifted so that f_0 = 0)
    maximum_iterations : int, self-consistent plus Newton iterations allowed before MBARConvergenceError
    relative_tolerance : float, convergence when max_i |g_i| / N_i over the sampled states is at most this
    """

    def __init__(self, u_kn, N_k, initial_f_k=None, maximum_iterations=10000, relative_tolerance=1.0e-12):
        self.u_kn = np.ascontiguousarray(u_kn, dtype=np.float64)
        self.N_k = np.asarray(N_k, dtype=np.int64).copy()
        if self.u_kn.ndim != 2 or self.N_k.shape != (self.u_kn.shape[0],):
            raise ValueError('u_kn must be (K, N) and N_k (K,)')
        if self.N_k.sum() != self.u_kn.shape[1]:
            raise ValueError('the samples N_k must add up to the columns of u_kn')
        if not np.all(np.isfinite(self.u_kn)):
            raise ValueError('u_kn must be finite')
        self._lib = _lib.load()
        h = C.c_void_p()
        K, N = self.u_kn.shape
        _check(self._lib, None, self._lib.rx_mbar_create(K, N, _ptr(self.u_kn), _ptr(self.N_k), C.byref(h)))
        self._start(h, initial_f_k, maximum_iterations, relative_tolerance)

    @classmethod
    def from_history(cls, engine, iterations, columns, N_k, initial_f_k=None, maximum_iterations=10000,
                     relative_tolerance=1.0e-12):
        """MBAR of u_kn gathered on the device from ``engine``'s energy history (Engine.history_append), with no host
        copy: row i of u_kn is history column ``columns[i]`` (the sampled states 0..M-1, then the unsampled ones), and
        column r * n + j is replica r at iteration ``iterations[j]``, n = len(iterations).  ``u_kn`` is None."""
        self = cls.__new__(cls)
        self.u_kn = None
        it = np.ascontiguousarray(iterations, dtype=np.int64)
        cols = np.ascontiguousarray(columns, dtype=np.int32)
        self.N_k = np.asarray(N_k, dtype=np.int64).copy()
        if it.ndim != 1 or cols.ndim != 1 or self.N_k.shape != cols.shape:
            raise ValueError('iterations and columns must be 1-D, and N_k as long as columns')
        self._lib = _lib.load()
        h = C.c_void_p()
        _check(self._lib, None, self._lib.rx_mbar_create_from_history(engine._h, len(cols), len(it), _ptr(it), _ptr(cols),
                                                                       _ptr(self.N_k), C.byref(h)))
        self._start(h, initial_f_k, maximum_iterations, relative_tolerance)
        return self

    def _start(self, h, initial_f_k, maximum_iterations, relative_tolerance):
        self._h = h
        self.n_iterations = 0
        try:
            self.f_k = self._solve(initial_f_k, int(maximum_iterations), float(relative_tolerance))
        except BaseException:
            self.close()
            raise
        self._theta = None

    def close(self):
        """Release the device copy of u_kn."""
        if getattr(self, '_h', None):
            self._lib.rx_mbar_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    # -- device calls
    def _evaluate(self, f, hessian):
        """(sum_n log D_n, gradient, Hessian or None, log sum_n W_in) at f."""
        K = len(f)
        f = np.ascontiguousarray(f, dtype=np.float64)
        s = C.c_double()
        g, lw = np.empty(K), np.empty(K)
        H = np.empty((K, K)) if hessian else None
        _check(self._lib, self._h, self._lib.rx_mbar_evaluate(self._h, _ptr(f), C.byref(s), _ptr(g),
                                                               _ptr(H) if hessian else None))
        _check(self._lib, self._h, self._lib.rx_mbar_get_log_wsum(self._h, _ptr(lw)))
        return s.value, g, H, lw

    def _gram(self, f):
        K = len(f)
        f = np.ascontiguousarray(f, dtype=np.float64)
        G, wsum = np.empty((K, K)), np.empty(K)
        _check(self._lib, self._h, self._lib.rx_mbar_gram(self._h, _ptr(f), _ptr(G), _ptr(wsum)))
        return G, wsum

    # -- solve
    def _solve(self, initial_f_k, maximum_iterations, tol):
        N = self.N_k.astype(np.float64)
        sampled = np.flatnonzero(self.N_k > 0)
        gauge = sampled[0]
        free = sampled[1:]                      # f[gauge] stays fixed during the solve
        f = np.zeros(len(N))
        if initial_f_k is not None:
            f[sampled] = np.asarray(initial_f_k, dtype=np.float64)[sampled]
            f -= f[gauge]
        f[self.N_k == 0] = 0.0

        def residual(lw):
            # |g_i| / N_i = |1 - sum_n W_in|, without the cancellation of 1 - sum when the sum is far from 1
            return np.max(np.abs(np.expm1(lw[sampled])))

        def floor(f):
            # exp's arguments f_i - u_in - log D_n are of the size of f, so each weight, and the residual, carries a
            # rounding error of about eps max|f|: a tolerance below that can only be met by chance
            return max(tol, 16.0 * np.finfo(np.float64).eps * np.max(np.abs(f[sampled])))

        # self-consistent iterations until the gradient is small enough for Newton steps
        it = 0
        while it < min(maximum_iterations, 50):
            logden, g, _, lw = self._evaluate(f, False)
            it += 1
            r = residual(lw)
            if r <= floor(f) or r < 1.0e-2:
                break
            f[sampled] -= lw[sampled]
            f[sampled] -= f[gauge]
        # Newton iterations on the log-likelihood, backtracking when a step lowers it
        logden, g, H, lw = self._evaluate(f, True)
        it += 1
        like = N @ f - logden
        while residual(lw) > floor(f):
            if it >= maximum_iterations:
                raise MBARConvergenceError('MBAR did not converge in %d iterations: relative gradient %.3g > %.3g'
                                           % (it, residual(lw), floor(f)))
            if len(free) == 0:
                break
            try:
                step = np.linalg.solve(H[np.ix_(free, free)], -g[free])
            except np.linalg.LinAlgError:
                step = np.full(len(free), np.nan)
            t = 1.0
            while np.all(np.isfinite(step)):
                trial = f.copy()
                trial[free] += t * step
                logden_t, g_t, H_t, lw_t = self._evaluate(trial, True)
                it += 1
                like_t = N @ trial - logden_t
                if like_t >= like - 1e-12 * abs(like) or it >= maximum_iterations:
                    break
                t *= 0.5
                if t < 1e-6:
                    step = step * np.nan
            if not np.all(np.isfinite(step)):
                # far from the solution a state whose weights all underflow makes H singular: a self-consistent
                # step, which is exact in log space at any distance, moves it instead
                trial = f.copy()
                trial[sampled] -= lw[sampled]
                trial[sampled] -= trial[gauge]
                logden_t, g_t, H_t, lw_t = self._evaluate(trial, True)
                it += 1
                like_t = N @ trial - logden_t
            f, g, H, like, lw = trial, g_t, H_t, like_t, lw_t
        self.n_iterations = it
        # states without samples: f_i = -log sum_n exp(-u_in) / D_n, from the last evaluation, which was at f_i = 0
        unsampled = self.N_k == 0
        f[unsampled] = -lw[unsampled]
        return f - f[0]

    # -- uncertainty
    def _covariance(self):
        if self._theta is None:
            G, _ = self._gram(self.f_k)
            s2, V = np.linalg.eigh(G)
            S = np.sqrt(np.clip(s2, 0.0, None))
            K = len(S)
            A = np.eye(K) - (S[:, None] * (V.T * self.N_k.astype(np.float64)) @ V * S[None, :])
            # A is singular along e = U^T 1_N = S^-1 V^T W^T 1_N = S^-1 V^T 1_K (W diag(N) W^T 1_N = 1_N and
            # W^T 1_N = 1_K at the solution).  A cutoff-based pseudo-inverse would keep or drop that direction by the
            # rounding of its eigenvalue, and keeping it adds a huge constant to Theta that cancels in dDelta_f only
            # to rounding; projecting it out exactly gives A^+ = (A + e e^T)^-1 - e e^T.
            e = np.divide(V.T @ np.ones(K), S, out=np.zeros(K), where=S > 0)
            e /= np.linalg.norm(e)
            VS = V * S[None, :]
            self._theta = VS @ (np.linalg.inv(A + np.outer(e, e)) - np.outer(e, e)) @ VS.T
        return self._theta

    def compute_free_energy_differences(self):
        """{'Delta_f': f_j - f_i, 'dDelta_f': its asymptotic standard deviation}, both (K, K) in kT."""
        f = self.f_k
        theta = self._covariance()
        d = np.diag(theta)
        var = d[:, None] + d[None, :] - 2.0 * theta
        return {'Delta_f': f[None, :] - f[:, None], 'dDelta_f': np.sqrt(np.clip(var, 0.0, None))}
