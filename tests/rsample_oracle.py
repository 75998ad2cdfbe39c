"""Float64 reference of the reparameterised sampler (b2b_chain_sample_logq_f32 / b2b_chain_sample_vjp_f32) on a given
base draw z: x = μ + σ ⊙ z or μ + L z, y = T(x),
    log q(y) = −½‖z‖² − Σ log σᵢ (or log Lᵢᵢ) − ½·D·log2π − ℓ(x),
and its reverse mode with z held fixed, composed from the chain oracle (chain_vjp_oracle.py)."""
import numpy as np

import chain_vjp_oracle as V

LOG2PI = float(np.log(2.0 * np.pi))


def base_x(z, mu=None, sigma=None, L=None, dtype=np.float64):
    z = np.asarray(z, dtype)
    x = np.asarray(L, dtype) @ z if L is not None else (z * np.asarray(sigma, dtype)[:, None] if sigma is not None else z)
    return x + np.asarray(mu, dtype)[:, None] if mu is not None else x


def base_logq(z, sigma=None, L=None, dtype=np.float64):
    z = np.asarray(z, dtype)
    D = z.shape[0]
    diag = np.diag(np.asarray(L, dtype)) if L is not None else (np.asarray(sigma, dtype) if sigma is not None else np.ones(D, dtype))
    return -0.5 * np.sum(z * z, axis=0) - np.sum(np.log(diag)) - 0.5 * D * LOG2PI


def forward(layers, flags, z, mu=None, sigma=None, L=None, dtype=np.float64):
    """(y, log q) of the chain `layers` (layer l inverted when flags[l]) over the base draw z."""
    x = base_x(z, mu, sigma, L, dtype)
    y, lj = V.chain_logjac(layers, flags, x, dtype=dtype) if layers else (x, np.zeros(x.shape[1], dtype))
    return y, base_logq(z, sigma, L, dtype) - lj


def vjp(layers, flags, z, ybar, qbar, mu=None, sigma=None, L=None, dtype=np.float64, x=None):
    """(per-layer cotangent dicts, base cotangents {"μ", "σ"} / {"μ", "L"} for the given parameters) of
    Σ ȳ·y + Σ q̄·log q with z fixed: x̄ from the chain's reverse mode with l̄ = −q̄, μ̄ = Σ x̄, σ̄ = Σ x̄ ⊙ z − Σq̄/σ,
    L̄ = tril(Σ x̄ zᵀ) − Σq̄·diag(1/Lᵢᵢ).  ``x`` (default: formed from z) is the point the chain is differentiated at:
    a device test passes the device's own base sample, so that both references see the same input as the device."""
    z = np.asarray(z, dtype)
    D, N = z.shape
    qb = np.zeros(N, dtype) if qbar is None else np.asarray(qbar, dtype)
    x = base_x(z, mu, sigma, L, dtype) if x is None else np.asarray(x, dtype)
    if layers:
        xb, grads, _ = V.chain_vjp(layers, flags, x, ybar, -qb, dtype=dtype)
    else:
        xb, grads = (np.zeros((D, N), dtype) if ybar is None else np.asarray(ybar, dtype)), []
    xb = np.asarray(xb, dtype)
    qs = qb.sum()
    base = {}
    if mu is not None:
        base["μ"] = xb.sum(axis=1)
    if L is not None:
        base["L"] = np.tril(xb @ z.T) - qs * np.diag(1.0 / np.diag(np.asarray(L, dtype)))
    elif sigma is not None:
        base["σ"] = (xb * z).sum(axis=1) - qs / np.asarray(sigma, dtype)
    return grads, base
