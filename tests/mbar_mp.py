"""MBAR at 50 significant digits in mpmath -- TEST INFRASTRUCTURE ONLY.

The exact MBAR quantities of a given float64 u_kn, for small problems (K <= 6, N <= 300): log D_n, log sum_n W_in, the
Gram matrix G = W^T W and the Hessian H at a given f; the solution f (self-consistent steps, then Newton); the
asymptotic covariance Theta and dDelta_f.  An mpf has an unbounded exponent, so exp(-u) of |u| ~ 1e6 kT is represented
as it is and nothing is shifted or taken in log space: this is the definition, evaluated with 50 digits.
"""
import mpmath as mp
import numpy as np

DPS = 50


class Reference:
    """MBAR of u_kn (K, N) float64 and N_k (K,) at DPS digits.  Every output is float64 except solve()'s."""

    def __init__(self, u_kn, N_k):
        u_kn = np.asarray(u_kn, dtype=np.float64)
        self.K, self.Nn = u_kn.shape
        self.N = [int(n) for n in N_k]
        self.sampled = [k for k in range(self.K) if self.N[k] > 0]
        with mp.workdps(DPS):
            # exp(-u_kn) once; D_n and W at any f need K exps more
            self.e = [[mp.exp(-mp.mpf(float(x))) for x in row] for row in u_kn]

    def _weights(self, f):
        """(log D_n [N], W [K][N]) at f (mpf list)."""
        ef = [mp.exp(x) for x in f]
        D = [mp.fsum(self.N[k] * ef[k] * self.e[k][n] for k in self.sampled) for n in range(self.Nn)]
        W = [[ef[i] * self.e[i][n] / D[n] for n in range(self.Nn)] for i in range(self.K)]
        return [mp.log(d) for d in D], W

    def evaluate(self, f):
        """{'logD', 'log_wsum', 'G', 'H', 'logden_sum'} at f, rounded to float64."""
        with mp.workdps(DPS):
            f = [mp.mpf(float(x)) for x in f]
            logD, W = self._weights(f)
            wsum = [mp.fsum(row) for row in W]
            G = [[mp.fsum(a * b for a, b in zip(W[i], W[j])) for j in range(self.K)] for i in range(self.K)]
            H = [[self.N[i] * self.N[j] * G[i][j] - (self.N[i] * wsum[i] if i == j else 0) for j in range(self.K)]
                 for i in range(self.K)]
            return {'logD': np.array([float(x) for x in logD]), 'log_wsum': np.array([float(mp.log(w)) for w in wsum]),
                    'G': np.array([[float(x) for x in r] for r in G]), 'H': np.array([[float(x) for x in r] for r in H]),
                    'logden_sum': float(mp.fsum(logD))}

    def solve(self, tol=mp.mpf(10) ** -40, max_iterations=500):
        """f (mpf list, f_0 = 0): self-consistent steps until |1 - sum_n W_in| < 1e-3, then Newton on the sampled
        states; states without samples from f_i = -log sum_n exp(-u_in) / D_n."""
        with mp.workdps(DPS):
            f = [mp.mpf(0)] * self.K
            g0, free = self.sampled[0], self.sampled[1:]
            for it in range(max_iterations):
                _, W = self._weights(f)
                wsum = [mp.fsum(row) for row in W]
                r = max(abs(1 - wsum[i]) for i in self.sampled)
                if r < tol:
                    break
                if r > mp.mpf('1e-3') or not free:
                    for i in self.sampled:
                        f[i] -= mp.log(wsum[i])
                else:
                    H = mp.matrix(len(free), len(free))
                    g = mp.matrix(len(free), 1)
                    for a, i in enumerate(free):
                        g[a] = self.N[i] - self.N[i] * wsum[i]
                        for b, j in enumerate(free):
                            H[a, b] = self.N[i] * self.N[j] * mp.fsum(x * y for x, y in zip(W[i], W[j])) - \
                                (self.N[i] * wsum[i] if i == j else 0)
                    step = mp.lu_solve(H, -g)
                    for a, i in enumerate(free):
                        f[i] += step[a]
                f = [x - f[g0] if self.N[k] > 0 else x for k, x in enumerate(f)]
            else:
                raise RuntimeError('mpmath MBAR did not converge: %s' % mp.nstr(r, 5))
            f = [x if self.N[k] > 0 else mp.mpf(0) for k, x in enumerate(f)]
            _, W = self._weights(f)
            for k in range(self.K):
                if self.N[k] == 0:
                    f[k] = -mp.log(mp.fsum(W[k]))
            return [x - f[0] for x in f]

    def theta(self, f):
        """Theta = V S ((A + e e^T)^-1 - e e^T) S V^T, A = I - S V^T diag(N) V S, from G = V S^2 V^T at f (mpf)."""
        with mp.workdps(DPS):
            _, W = self._weights(f)
            K = self.K
            G = mp.matrix([[mp.fsum(a * b for a, b in zip(W[i], W[j])) for j in range(K)] for i in range(K)])
            s2, V = mp.eigsy(G)
            S = [mp.sqrt(max(x, 0)) for x in s2]
            VS = mp.matrix(K, K)
            for i in range(K):
                for j in range(K):
                    VS[i, j] = V[i, j] * S[j]
            A = mp.eye(K) - VS.T * mp.diag([mp.mpf(n) for n in self.N]) * VS
            e = V.T * mp.matrix([1] * K)
            for i in range(K):
                e[i] = e[i] / S[i] if S[i] > 0 else 0
            e = e / mp.norm(e)
            P = e * e.T
            return VS * (mp.inverse(A + P) - P) * VS.T

    def ddf(self, f):
        """dDelta_f (K, K) float64 at f (mpf)."""
        with mp.workdps(DPS):
            T = self.theta(f)
            return np.array([[float(mp.sqrt(max(T[i, i] + T[j, j] - 2 * T[i, j], 0))) for j in range(self.K)]
                             for i in range(self.K)])


# -- reduced potentials at the energy scales of real runs ---------------------------------------------------------------
def offsets(K, n_per, delta, seed, d=0.0, d_spread=0.0):
    """K states whose rows differ by offsets 0 .. delta kT on N(0, 1) noise, n_per samples each, every sample shifted by
    d + U(-d_spread, d_spread) kT."""
    rng = np.random.default_rng(seed)
    N = K * n_per
    u = rng.normal(0.0, 1.0, (K, N)) + np.linspace(0.0, delta, K)[:, None]
    u += d + rng.uniform(-d_spread, d_spread, N)[None, :]
    return u, np.full(K, n_per, np.int64)


KB = 0.008314462618      # kJ/mol/K


def temperature_ladder(n_atoms, T0, T1, K, n_per, seed, unsampled=0.0):
    """A parallel-tempering run's u_kn: potential energies of n_atoms atoms (-15 kJ/mol per atom plus a heat capacity
    of 1.5 k_B per atom, Gaussian at each temperature) sampled at K geometric temperatures T0..T1, n_per each, reduced
    as E / k_B T_k.  With unsampled != 0, two states without samples: the coldest state shifted down by `unsampled` kT
    first and the hottest shifted up by it last, whose f are exactly f_1 - unsampled and f_K + unsampled."""
    rng = np.random.default_rng(seed)
    T = T0 * (T1 / T0) ** (np.arange(K) / max(K - 1, 1))
    E = np.concatenate([n_atoms * (-15.0 + 1.5 * KB * t) + rng.normal(0.0, KB * t * np.sqrt(1.5 * n_atoms), n_per)
                        for t in T])
    u = E[None, :] / (KB * T[:, None])
    N_k = np.full(K, n_per, np.int64)
    if unsampled:
        u = np.concatenate([u[:1] - unsampled, u, u[-1:] + unsampled])
        N_k = np.r_[0, N_k, 0]
    return u, N_k
