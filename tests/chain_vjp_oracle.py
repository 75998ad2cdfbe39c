"""Float64 restatements of the reverse mode of the elementwise layers (Stacked laws, Permute), of the terminal MvNormal and
of whole mixed chains of every layer kind, closed by either terminal -- the references of b2b_chain_vjp_f32.  They
compose the per-kind VJPs of oracle/oracle_np.py and of the spline / MLP coupling and dense Scale references, and are
themselves checked against central finite differences (tests/test_oracle_chain_vjp.py)."""
from __future__ import annotations

import numpy as np

import mvnormal_tril_oracle as T
from oracle import oracle_np as O

EW = O.EW


def _law_deriv(op, inverse, x):
    """(f′, ∂log|f′|/∂x) of one Stacked law at x (float64): what AD of the reference's formulas gives, including
    _clamp's zero derivative outside [lb, ub] (Bijectors.jl:95-100) and LeakyReLU's identity branch at 0."""
    code = op[0]
    a = float(op[1]) if len(op) > 1 else 0.0
    b = float(op[2]) if len(op) > 2 else 0.0
    one, zero = np.ones_like(x), np.zeros_like(x)
    if code in (EW.EXP, EW.LOG):
        if (code == EW.EXP) != inverse:
            return np.exp(x), one
        return 1 / x, -1 / x
    if code == EW.SCALE:
        return one * (1 / a if inverse else a), zero
    if code == EW.LEAKY_RELU:
        al = 1 / a if inverse else a
        return np.where(x < 0, al, 1.0), zero
    if code == EW.LOGIT:
        if not inverse:
            return 1 / (x - a) + 1 / (b - x), 1 / (b - x) - 1 / (x - a)
        s = O._logistic(x)
        return (b - a) * s * (1 - s), 1 - 2 * s
    if code == EW.TRUNCATED:
        lo, hi = np.isfinite(a), np.isfinite(b)
        if not inverse:
            inside = (x >= a) & (x <= b)
            xc = np.where(inside, x, (a if lo else 0.0) + 0.5)  # any interior point: the result is masked
            if lo and hi:
                f, d = 1 / (xc - a) + 1 / (b - xc), 1 / (b - xc) - 1 / (xc - a)
            elif lo:
                f, d = 1 / (xc - a), -1 / (xc - a)
            elif hi:
                f, d = -1 / (b - xc), 1 / (b - xc)
            else:
                f, d = one, zero
            return np.where(inside, f, 0.0), np.where(inside, d, 0.0)
        if lo and hi:
            s = O._logistic(x)
            xo, f, d = (b - a) * s + a, (b - a) * s * (1 - s), 1 - 2 * s
        elif lo or hi:
            e = np.exp(x)
            xo, f, d = (e + a if lo else b - e), (e if lo else -e), one
        else:
            xo, f, d = x, one, zero
        return np.where((xo < a) | (xo > b), 0.0, f), d
    return one, zero  # IDENTITY, SHIFT


def stacked_vjp(ops, ranges, x, ybar, ljbar, inverse=False):
    """Input cotangent of with_logabsdet_jacobian(Stacked(laws, ranges), x) (or of its inverse): x̄ = ȳ·f′ + l̄·∂log|f′|/∂x
    per element.  ``ops`` / ``ranges`` as in oracle_np.stacked_forward; x, ybar (D, N), ljbar (N,)."""
    x = np.asarray(x)
    xbar = np.empty_like(x)
    lb = np.asarray(ljbar, x.dtype)[None, :]
    for op, (lo, hi) in zip(ops, ranges):
        f, d = _law_deriv(op, inverse, x[lo - 1:hi])
        xbar[lo - 1:hi] = ybar[lo - 1:hi] * f + lb * d
    return xbar


def permute_vjp(A, ybar, inverse=False):
    """Input cotangent of Permute(A) (y = A x, permute.jl:152) or of its inverse (x = Aᵀ y, :153): Aᵀ ȳ or A x̄."""
    A = np.asarray(A, np.float64)
    return (A @ ybar) if inverse else (A.T @ ybar)


def mvnormal_diag_logpdf_vjp(mu, sigma, x, lpbar):
    """Cotangents (x̄, μ̄, σ̄) of logpdf(MvNormal(μ, Diagonal(σ²)), x) with cotangent lpbar (N,) of the logpdf vector:
    q = (x − μ)/σ, x̄ = −l̄·q/σ, μ̄ = Σ_n l̄·q/σ, σ̄ = Σ_n l̄·(q² − 1)/σ."""
    x = np.asarray(x)
    D, dt = x.shape[0], x.dtype
    mu = np.zeros(D, dt) if mu is None else np.asarray(mu, dt)
    sigma = np.ones(D, dt) if sigma is None else np.asarray(sigma, dt)
    q = (x - mu[:, None]) / sigma[:, None]
    lb = np.asarray(lpbar, dt)[None, :]
    g = lb * q / sigma[:, None]
    return -g, g.sum(axis=1), (lb * (q * q - 1) / sigma[:, None]).sum(axis=1)


def _layer_vjp(lay, inv: bool, x, ybar, ljbar, b_terms=None):
    """(x̄, parameter cotangents as a dict keyed like the device grads) of one oracle layer applied to x: an O.Layer, or a
    SplineLayer / MLPLayer / ScaleLayer, whose own .vjp evaluates in x's dtype.  A planar layer appends the N column
    terms of its b̄ to the list ``b_terms`` when one is given."""
    k = lay.kind
    if k in ("coupling_rqs", "coupling_mlp", "scale_matrix"):
        return lay.vjp(x, ybar, ljbar, inverse=inv)
    p = lay.params
    if k == "planar":
        fn = O.planar_inverse_chain_vjp if inv else O.planar_chain_vjp
        xb, g = fn([(p["w"], p["u"], p["b"])], x, ybar, ljbar, b_terms=b_terms)
        return xb, dict(w=g[0][0], u=g[0][1], b=g[0][2])
    if k == "radial":
        xb, g = O.radial_chain_vjp_dir([(p["alpha_raw"], p["beta"], p["z0"])], [inv], x, ybar, ljbar)
        return xb, {"α_": g[0][0], "β": g[0][1], "z_0": g[0][2]}
    if k == "rqs":
        xb, W, H, Dv = O.rqs_vjp(p["widths"], p["heights"], p["derivs"], x, ybar, ljbar, inverse=inv)
        return xb, dict(widths=W, heights=H, derivatives=Dv)
    if k == "coupling_affine":
        xb, W, c = O.coupling_affine_vjp(p["idx1"], p["idx2"], p["W"], p["c"], x, ybar, ljbar, inverse=inv)
        return xb, dict(W=W, c=c)
    if k == "batchnorm":
        xb, b, ls = O.batchnorm_eval_vjp(p["bn"], x, ybar, ljbar, inverse=inv)
        return xb, dict(b=b, logs=ls)
    if k == "permute":
        return permute_vjp(p["A"], ybar, inverse=inv), {}
    if k == "stacked":
        return stacked_vjp(p["ops"], p["ranges"], x, ybar, ljbar, inverse=inv), {}
    raise ValueError(k)


def chain_vjp(layers, inverse_flags, x, ybar, ljbar, mu=None, sigma=None, terminal=False, dtype=np.float64,
              scale_tril=None, b_terms=None):
    """Reverse mode of a chain applied in the given order (layer l inverted when inverse_flags[l]), optionally closed by
    a terminal MvNormal (then the log-Jacobian output is logpdf): MvNormal(μ, Diagonal(σ²)) when ``terminal``, or
    MvNormal(μ, L Lᵀ) when ``scale_tril`` = L is given.  ybar (D, N) or None (zeros), ljbar (N,) or None (zeros).
    Evaluated in `dtype` (float32 gives the reference's own float32 error for the parity gate).
    Returns (x̄, [grads dict per layer], the base's cotangents: {"μ": …, "σ": …} / {"μ": …, "L": …}, μ̄ and σ̄ only for
    a given μ / σ; {} without a terminal).  A dict ``b_terms`` receives {l: the N column terms of b̄} for every planar
    layer l, whose sum is that layer's b̄."""
    x = np.asarray(x, dtype)
    N = x.shape[1]
    lb = np.zeros(N, dtype) if ljbar is None else np.asarray(ljbar, dtype)
    inputs, cur = [], x
    for lay, inv in zip(layers, inverse_flags):
        inputs.append(cur)
        cur = (lay.inverse if inv else lay.forward)(cur)[0]
    g = np.zeros_like(cur) if ybar is None else np.asarray(ybar, dtype)
    base = {}
    if scale_tril is not None:
        gx, gm, gL = T.logpdf_vjp(scale_tril, mu, cur, lb, dtype)
        g = g + gx
        if mu is not None:
            base["μ"] = gm
        base["L"] = gL
    elif terminal:
        mu_, sigma_ = (None if v is None else np.asarray(v, dtype) for v in (mu, sigma))
        gx, gm, gs = mvnormal_diag_logpdf_vjp(mu_, sigma_, cur, lb)
        g = g + gx
        if mu is not None:
            base["μ"] = gm
        if sigma is not None:
            base["σ"] = gs
    grads = [None] * len(layers)
    for l in reversed(range(len(layers))):
        terms = [] if b_terms is not None and layers[l].kind == "planar" else None
        g, grads[l] = _layer_vjp(layers[l], inverse_flags[l], inputs[l], g, lb, terms)
        if terms:
            b_terms[l] = terms[0]
    return g, grads, base


def chain_logjac(layers, inverse_flags, x, mu=None, sigma=None, terminal=False, dtype=np.float64, scale_tril=None):
    """(y, logjac or logpdf) of the same chain, in `dtype` (float64 for finite differences and references, float32 for
    the reference's own error); the terminal as in chain_vjp."""
    cur, lj = np.asarray(x, dtype), 0.0
    for lay, inv in zip(layers, inverse_flags):
        cur, l = (lay.inverse if inv else lay.forward)(cur)
        lj = lj + l
    if scale_tril is not None:
        lj = lj + T.logpdf(scale_tril, mu, cur, dtype)
    elif terminal:
        lj = lj + O.mvnormal_diag_logpdf(*(None if v is None else np.asarray(v, dtype) for v in (mu, sigma)), cur)
    return cur, np.asarray(lj, dtype)
