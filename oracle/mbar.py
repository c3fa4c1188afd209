"""Independent MBAR in numpy / scipy (Shirts & Chodera 2008) -- TEST INFRASTRUCTURE ONLY.

The free energies solve the MBAR equations sum_n W_in = 1 for every sampled state i, with
W_in = exp(f_i - u_in) / sum_k N_k exp(f_k - u_kn); scipy's root finder solves them for the sampled states with f_0 = 0
(the first sampled state during the solve), states without samples follow from the same equation.  The sums over
samples are taken in log space (log_wsum), and solve shifts each sample by its lowest sampled energy first, which leaves
f unchanged: states thousands of kT apart and |u| ~ 1e5 kT are solved to rounding.  The covariance is
the asymptotic one, Theta = W^T (I - W diag(N) W^T)^+ W, taken as V S (I - S V^T diag(N) V S)^+ S V^T from the SVD
W = U S V^T of the weight matrix itself."""
import numpy as np
from scipy import optimize
from scipy.special import logsumexp


def log_denominator(u_kn, N_k, f_k):
    """log D_n = logsumexp_k (log N_k + f_k - u_kn), over the states with samples."""
    s = np.asarray(N_k) > 0
    return logsumexp(np.log(np.asarray(N_k, float)[s])[:, None] + np.asarray(f_k)[s, None] - u_kn[s], axis=0)


def weights(u_kn, N_k, f_k):
    """W (N x K): W_nk = exp(f_k - u_kn - log D_n)."""
    return np.exp(np.asarray(f_k)[:, None] - u_kn - log_denominator(u_kn, N_k, f_k)[None, :]).T


def log_wsum(u_kn, N_k, f_k):
    """log sum_n W_in = logsumexp_n (f_i - u_in - log D_n), finite at any energy scale."""
    return logsumexp(np.asarray(f_k)[:, None] - u_kn - log_denominator(u_kn, N_k, f_k)[None, :], axis=1)


def shift_samples(u_kn, N_k):
    """u_kn - m_n with m_n = min over the sampled states of u_kn: the same MBAR f and W, smaller exp arguments."""
    return u_kn - u_kn[np.asarray(N_k) > 0].min(axis=0)[None, :]


def evaluate(u_kn, N_k, f_k):
    """(sum_n log D_n, gradient g_i = N_i - N_i sum_n W_in, Hessian N_i N_j (W^T W)_ij - delta_ij N_i sum_n W_in,
    W^T W, sum_n W_in, log D_n) of the log-likelihood sum_k N_k f_k - sum_n log D_n."""
    N = np.asarray(N_k, float)
    logD = log_denominator(u_kn, N_k, f_k)
    W = np.exp(np.asarray(f_k)[:, None] - u_kn - logD[None, :]).T
    wsum = W.sum(axis=0)
    G = W.T @ W
    H = N[:, None] * N[None, :] * G - np.diag(N * wsum)
    return logD.sum(), N - N * wsum, H, G, wsum, logD


def solve(u_kn, N_k, tol=1e-13):
    """f_k (f_0 = 0) from scipy.optimize.root on the MBAR equations of the sampled states."""
    u_kn = shift_samples(np.asarray(u_kn, float), N_k)
    N = np.asarray(N_k, float)
    K = len(N)
    sampled = np.flatnonzero(N > 0)
    free = sampled[1:]
    f = np.zeros(K)
    for _ in range(20):       # a few self-consistent steps as the starting point
        f[sampled] -= log_wsum(u_kn, N_k, f)[sampled]
        f[sampled] -= f[sampled[0]]

    def eqs(x):
        # -g_i / N_i = expm1(log sum_n W_in) and the Hessian's rows / N_i, over the free states
        y = f.copy()
        y[free] = x
        a = y[free, None] - u_kn[free] - log_denominator(u_kn, N_k, y)[None, :]
        lw, W = logsumexp(a, axis=1), np.exp(a)
        H = N[free, None] * N[None, free] * (W @ W.T) - np.diag(N[free] * np.exp(lw))
        return -np.expm1(lw), H / N[free, None]

    if len(free):
        sol = optimize.root(eqs, f[free], jac=True, method='hybr', options={'xtol': 1e-15})
        f[free] = sol.x
    unsampled = N == 0
    if unsampled.any():
        f0 = f.copy()
        f0[unsampled] = 0.0
        f[unsampled] = -log_wsum(u_kn, N_k, f0)[unsampled]
    f = f - f[0]
    err = np.max(np.abs(np.expm1(log_wsum(u_kn, N_k, f)[sampled])))
    if err > tol * 100:
        raise RuntimeError('oracle MBAR did not converge: %g' % err)
    return f


def covariance(u_kn, N_k, f_k):
    W = weights(u_kn, N_k, f_k)
    U, S, Vt = np.linalg.svd(W, full_matrices=False)
    V = Vt.T
    K = len(S)
    A = np.eye(K) - (S[:, None] * (Vt * np.asarray(N_k, float)[None, :]) @ V * S[None, :])
    # A is singular along U^T 1_N (W diag(N) W^T 1_N = 1_N at the solution); its pseudo-inverse projects that out
    e = U.T @ np.ones(len(U))
    e /= np.linalg.norm(e)
    VS = V * S[None, :]
    return VS @ (np.linalg.inv(A + np.outer(e, e)) - np.outer(e, e)) @ VS.T


def free_energy_differences(u_kn, N_k):
    """(Delta_f_ij = f_j - f_i, dDelta_f_ij) in kT."""
    f = solve(u_kn, N_k)
    theta = covariance(shift_samples(np.asarray(u_kn, float), N_k), N_k, f)
    d = np.diag(theta)
    return f[None, :] - f[:, None], np.sqrt(np.clip(d[:, None] + d[None, :] - 2 * theta, 0, None)), f
