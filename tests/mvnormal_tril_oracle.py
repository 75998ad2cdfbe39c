"""Float64 reference for the full-covariance MvNormal base, B2B_MVNORMAL_TRIL: MvNormal(μ, Σ) with Σ = L Lᵀ
(Distributions' FullNormal; PDMats holds the Cholesky factor L).  With δ = x − μ, r = L⁻¹δ and s = L⁻ᵀr:

    logpdf(x) = −½·D·log2π − Σᵢ log Lᵢᵢ − ½·rᵀr
    rand      = μ + L z
    x̄ = ȳ − l̄·s,   μ̄ = Σₙ l̄ₙ sₙ,   L̄ = tril(Σₙ l̄ₙ sₙ rₙᵀ) − (Σₙ l̄ₙ)·diag(1/Lᵢᵢ)

Every function takes a ``dtype``: float32 evaluates the same formulas in float32 (LAPACK's strtrs), which gives the
reference's own float32 error for the parity gates.  Whole chains closed by this terminal are chain_vjp_oracle's
chain_logjac / chain_vjp with ``scale_tril``."""
import math

import numpy as np
from scipy.linalg import solve_triangular


def _prep(L, mu, x, dtype):
    dt = np.dtype(dtype)
    L = np.tril(np.asarray(L, dt))
    x = np.asarray(x, dt)
    d = x if mu is None else x - np.asarray(mu, dt)[:, None]
    return dt, L, d


def logpdf(L, mu, x, dtype=np.float64):
    """logpdf(MvNormal(μ, L Lᵀ), x) for x (D, N); ``mu`` may be None (zeros)."""
    dt, L, d = _prep(L, mu, x, dtype)
    r = solve_triangular(L, d, lower=True)
    c = dt.type(-0.5 * L.shape[0] * math.log(2 * math.pi)) - np.sum(np.log(np.diag(L)), dtype=dt)
    return (c - dt.type(0.5) * np.sum(r * r, axis=0, dtype=dt)).astype(dt)


def logpdf_vjp(L, mu, x, lpbar, dtype=np.float64):
    """(−l̄·s (D, N): the logpdf's share of x̄, μ̄ (D,), L̄ (D, D) lower triangular)."""
    dt, L, d = _prep(L, mu, x, dtype)
    lb = np.asarray(lpbar, dt)
    r = solve_triangular(L, d, lower=True)
    s = solve_triangular(L, r, lower=True, trans="T")
    ls = lb[None, :] * s
    Lbar = np.tril(ls @ r.T) - np.sum(lb, dtype=dt) * np.diag(dt.type(1) / np.diag(L))
    return (-ls).astype(dt), ls.sum(axis=1).astype(dt), Lbar.astype(dt)


def sample(L, mu, z):
    """μ + L z for base normals z (D, N)."""
    L = np.tril(np.asarray(L, np.float64))
    y = L @ np.asarray(z, np.float64)
    return y if mu is None else y + np.asarray(mu, np.float64)[:, None]


def random_tril(rng, D, cond=1.0, dtype=np.float64):
    """A lower factor with positive diagonal; ``cond`` > 1 scales its columns by factors spread over [1/cond, 1], so that
    L is ill-conditioned (condition number ≳ cond)."""
    L = np.tril(rng.standard_normal((D, D))) * (0.5 / math.sqrt(D))
    L[np.arange(D), np.arange(D)] = rng.uniform(0.7, 1.3, D)
    if cond > 1:
        L = L * np.exp(rng.uniform(-math.log(cond), 0.0, D))[None, :]
    return L.astype(dtype)
