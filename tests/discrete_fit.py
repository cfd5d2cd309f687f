"""Goodness-of-fit helpers of the discrete-sampler tests."""

import numpy as np
import scipy.stats as st


def chi2_pvalue(x, dist, bins=200):
    """Chi-squared goodness of fit of integer draws `x` against a frozen scipy discrete distribution: cut points at the
    distribution's quantiles, tail bins pooled, and neighbouring bins merged until every expected count is at least 5."""
    x = np.asarray(x)
    n = x.size
    q = np.linspace(0.0, 1.0, min(bins, max(2, n // 20)) + 1)[1:-1]
    cuts = np.unique(np.floor(dist.ppf(q)))
    cdf = np.concatenate([[0.0], dist.cdf(cuts), [1.0]])
    expected = n * np.diff(cdf)
    observed = np.bincount(np.searchsorted(cuts, x, side="left"), minlength=cuts.size + 1).astype(np.float64)
    return chi2_counts(observed, expected)


def chi2_counts(observed, expected):
    """Chi-squared p-value of observed category counts against expected ones, neighbouring categories merged until every
    expected count is at least 5."""
    n = float(np.sum(observed))
    e, o = [], []
    ce = co = 0.0
    for ei, oi in zip(expected, observed):
        ce += ei
        co += oi
        if ce >= 5.0:
            e.append(ce)
            o.append(co)
            ce = co = 0.0
    if ce or co:
        if e:
            e[-1] += ce
            o[-1] += co
        else:
            e, o = [ce], [co]
    e, o = np.array(e), np.array(o)
    if e.size < 2:
        return 1.0 if o.sum() == n else 0.0
    return float(st.chisquare(o, e * (o.sum() / e.sum())).pvalue)


def moments_ok(x, mean, var, k=5.0):
    """Sample mean and variance within k standard errors (the variance's from the sample's own fourth moment)."""
    x = np.asarray(x, dtype=np.float64)
    n = x.size
    m4 = np.mean((x - x.mean()) ** 4)
    ok_mean = abs(x.mean() - mean) <= k * np.sqrt(var / n) + 1e-12 * abs(mean)
    ok_var = abs(x.var() - var) <= k * np.sqrt(max(m4 - var * var, 0.0) / n) + 1e-12 * var
    return bool(ok_mean and ok_var), (x.mean(), mean, x.var(), var)
