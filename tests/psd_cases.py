"""Graphs and inputs shared by the CPU and GPU tests of the Cholesky-solve nodes: a Gaussian-process marginal likelihood
(ExpQuad kernel + noise), its predictive mean and covariance, and a batched multivariate-normal log-density.  Written the
usual way (cholesky + two solve_triangular); PyTensor's rewrites turn the paired solves into CholeskySolve and the Cholesky
gradient of a batch into Blockwise(AllocDiag)."""

import numpy as np

import pytensor.tensor as pt


def _exp_quad(X1, X2, ell, eta):
    d2 = pt.sum((X1[:, None, :] - X2[None, :, :]) ** 2, axis=-1)
    return eta**2 * pt.exp(-0.5 * d2 / ell**2)


def gp_graph():
    """(inputs, [logp, d logp / d(ell, eta, sigma), predictive mean, predictive covariance])."""
    X, Xs = pt.dmatrix("X"), pt.dmatrix("Xs")
    y = pt.dvector("y")
    ell, eta, sigma = pt.dscalar("ell"), pt.dscalar("eta"), pt.dscalar("sigma")
    n = X.shape[0]
    K = _exp_quad(X, X, ell, eta) + sigma**2 * pt.eye(n)
    L = pt.linalg.cholesky(K)
    alpha = pt.linalg.solve_triangular(L.T, pt.linalg.solve_triangular(L, y, lower=True), lower=False)
    logp = -0.5 * pt.dot(y, alpha) - pt.sum(pt.log(pt.diagonal(L))) - 0.5 * n * np.log(2 * np.pi)
    grads = pt.grad(logp, [ell, eta, sigma])
    Ks = _exp_quad(X, Xs, ell, eta)
    v = pt.linalg.solve_triangular(L, Ks, lower=True)
    mean = pt.dot(Ks.T, alpha)
    cov = _exp_quad(Xs, Xs, ell, eta) - pt.dot(v.T, v)
    return [X, Xs, y, ell, eta, sigma], [logp, *grads, mean, cov]


def gp_inputs(n, m, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 10, (n, 2))
    Xs = rng.uniform(0, 10, (m, 2))
    y = np.sin(X[:, 0]) + 0.3 * np.cos(2 * X[:, 1]) + 0.1 * rng.standard_normal(n)
    return [X, Xs, y, np.float64(1.3 + 0.2 * rng.random()), np.float64(0.9 + 0.2 * rng.random()),
            np.float64(0.3 + 0.1 * rng.random())]


def mvn_graph():
    """Batched MvNormal log-density summed over the batch, and its gradient w.r.t. mu and Sigma."""
    x, mu = pt.dmatrix("x"), pt.dmatrix("mu")
    S = pt.dtensor3("S")
    L = pt.linalg.cholesky(S)
    z = pt.linalg.solve_triangular(L, x - mu, lower=True, b_ndim=1)
    k = x.shape[-1]
    logp = pt.sum(-0.5 * pt.sum(z**2, axis=-1) - pt.sum(pt.log(pt.diagonal(L, axis1=-2, axis2=-1)), axis=-1)
                  - 0.5 * k * np.log(2 * np.pi))
    return [x, mu, S], [logp, *pt.grad(logp, [mu, S])]


def mvn_inputs(B, n, seed):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((B, n, n))
    S = M @ M.transpose(0, 2, 1) / n + np.eye(n)
    return [rng.standard_normal((B, n)), 0.1 * rng.standard_normal((B, n)), S]


def spd(rng, n, batch=(), dtype="float64"):
    M = rng.standard_normal(batch + (n, n))
    return (M @ np.swapaxes(M, -1, -2) / n + np.eye(n)).astype(dtype)
