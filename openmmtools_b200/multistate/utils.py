"""Exceptions and timeseries helpers of the multistate package (openmmtools/multistate/utils.py:51,
:107-193, :234-297).

The statistical inefficiency is restated from its definition (Chodera 2016, J. Chem. Theory Comput. 12, 1799):
g = 1 + 2 sum_{t>=1} (1 - t/T) C_t with C_t the normalised autocorrelation of the series at lag t, the sum stopping at the
first C_t <= 0 past a minimum lag of 3; with ``fast`` the lag advances by 1, 2, 3, ... and each term counts for the
lags it skips."""
import numpy as np


class SimulationNaNError(Exception):
    """Error when a simulation goes to NaN."""
    pass


def statistical_inefficiency_multiple(series, fast=False, mintime=3):
    """Statistical inefficiency g >= 1 of one or more timeseries of one process (a list of 1-D arrays, or a 2-D array
    of rows); the mean, variance and autocorrelation are pooled over the series.  Raises ValueError when the pooled
    series has zero variance."""
    rows = [np.asarray(s, dtype=np.float64).ravel() for s in series]
    lengths = np.array([len(r) for r in rows])
    total = np.concatenate(rows)
    mu = total.mean()
    d = [r - mu for r in rows]
    sigma2 = np.mean((total - mu) ** 2)
    if sigma2 == 0:
        raise ValueError('statistical inefficiency of a series with zero variance is undefined')
    T = lengths.mean()
    g, t, inc = 1.0, 1, 1
    while t < lengths.max() - 1:
        num = sum(float(np.dot(x[:len(x) - t], x[t:])) for x in d if len(x) > t)
        den = float(np.sum(np.clip(lengths - t, 0, None)))
        C = num / den / sigma2
        if C <= 0.0 and t > mintime:
            break
        g += 2.0 * C * (1.0 - t / T) * inc
        t += inc
        if fast:
            inc += 1
    return max(g, 1.0)


def statistical_inefficiency(series, fast=False, mintime=3):
    """Statistical inefficiency g >= 1 of one 1-D timeseries (see the module docstring)."""
    return statistical_inefficiency_multiple([series], fast=fast, mintime=mintime)


def subsample_correlated_data(series, g):
    """Indices of the roughly independent samples of a series of statistical inefficiency g: round(n g), n = 0, 1, ...,
    without repeats."""
    T = len(series)
    out, n = [], 0
    while int(round(n * g)) < T:
        t = int(round(n * g))
        if not out or t != out[-1]:
            out.append(t)
        n += 1
    return out


def get_equilibration_data_per_sample(timeseries_to_analyze, fast=True, max_subset=100):
    """For up to ``max_subset`` evenly spaced origins t of the series: (t, g of the series from t, effective samples
    (T - t + 1) / g), without the first origin (utils.py:107-193)."""
    series = np.array(timeseries_to_analyze)
    size = series.size
    n = size - 1
    if max_subset is None or n < max_subset:
        max_subset = n
    if max_subset == 0:
        max_subset = 1
    if series.std() == 0.0 or max_subset == 1:
        return np.arange(max_subset, dtype=int), np.array([1] * max_subset), np.arange(size, size - max_subset, -1)
    i_t = np.floor(np.arange(max_subset) * size / max_subset).astype(int)
    g_i = np.ones(max_subset, np.float32)
    n_effective_i = np.ones(max_subset, np.float32)
    for i, t in enumerate(i_t):
        g_i[i] = statistical_inefficiency(series[t:], fast=fast)
        n_effective_i[i] = (size - t + 1) / g_i[i]
    return i_t[1:], g_i[1:], n_effective_i[1:]


def remove_unequilibrated_data(data, number_equilibrated, axis):
    """``data`` without its first ``number_equilibrated`` entries along ``axis``."""
    data = np.asarray(data)
    index = [slice(None)] * data.ndim
    index[axis] = slice(number_equilibrated, None)
    return data[tuple(index)]


def subsample_data_along_axis(data, subsample_rate, axis):
    """``data`` at the indices subsample_correlated_data picks for statistical inefficiency ``subsample_rate``."""
    data = np.asarray(data)
    return np.take(data, subsample_correlated_data(np.zeros(data.shape[axis]), subsample_rate), axis=axis)
