"""CPU ORACLE (test infrastructure, NOT product code) -- numpy restatement of the Bijectors.jl hot path.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` leg may
import this module.  The product path (``bijectors.jl_b200``) never imports it and never falls back to it.

Every function follows the reference source line by line (citations are ``path:line`` relative to the
reference checkout, Bijectors.jl v0.16.2).  The reference is pure Julia and no Julia toolchain exists in
the build container, so the reference itself cannot be executed here: this restatement is pinned by

  * the deterministic golden vectors the reference's own tests hold (``tests/golden/reference_vectors.json``,
    transcribed from test/bijectors/{coupling,permute,stacked,rational_quadratic_spline}.jl,
    test/normalising_flows.jl and the doctest at src/interface.jl:21-31), checked in
    ``tests/test_oracle_golden.py``;
  * the reference's property tests restated in ``tests/test_oracle_properties.py`` (logjac vs. the
    log|det| of a numerical Jacobian, inverse∘forward = id, ``ires == (x, -logjac)``, the find_alpha
    residual grid of test/normalising_flows.jl:47-71).

Values in the reference tests that depend on Julia RNG streams (``randn`` after ``seed!``, ``StableRNG``)
are NOT reproducible without Julia: for those inputs parity is "pinned by property, not by value".

Arithmetic that lives in third-party Julia packages (not in the reference repository; no Manifest is vendored,
only compat ranges in Project.toml) is restated from its published maths:
  LogExpFunctions (compat 0.3.3, 1.0)  log1pexp, softmax
  Roots (compat 1.3.15, 2, 3)          find_zero(..., A42()) -> any bracketing solver converging to
                                        adjacent floats is admissible (results are pinned by the residual)
  ChangesOfVariables 0.1                with_logabsdet_jacobian of ComposedFunction / Fix1{broadcast}
  InverseFunctions 0.1                  inverse(f∘g) = inverse(g)∘inverse(f)
  Distributions 0.25.33 + PDMats        logpdf(MvNormal(mu, Diagonal), x)

Layout convention: a Julia ``D×N`` column-major matrix is a numpy array of shape ``(D, N)`` here
(numpy keeps Julia's index semantics; memory order is irrelevant for the oracle).
All functions compute in the dtype of their inputs (float32 in -> float32 arithmetic, like Julia).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

# --------------------------------------------------------------------------------------------------
# third-party scalar functions (SURVEY Appendix A.0)
# --------------------------------------------------------------------------------------------------


def log1pexp(x):
    """LogExpFunctions.log1pexp: numerically stable log(1 + exp(x)) (softplus).

    Restated from the documented maths: log1p(exp(x)) for x <= 0 and x + log1p(exp(-x)) for x > 0,
    which agrees with the package's 4-branch form to < 1 ulp.  Call sites: src/bijectors/planar_layer.jl:67-68,
    src/bijectors/radial_layer.jl:44-45,77-78,91-92, src/bijectors/rational_quadratic_spline.jl:105,116.
    """
    x = np.asarray(x)
    dt = x.dtype if x.dtype.kind == "f" else np.float64
    x = x.astype(dt, copy=False)
    with np.errstate(over="ignore"):
        out = np.where(x > 0, x + np.log1p(np.exp(-np.abs(x))), np.log1p(np.exp(-np.abs(x))))
    return out.astype(dt)[()]


def softmax_rows(v):
    """LogExpFunctions.softmax(v; dims=2): exp(v - max) / sum(exp(v - max)) along each row.

    Call site: src/bijectors/rational_quadratic_spline.jl:103-104,112-113.
    """
    v = np.asarray(v)
    m = v.max(axis=-1, keepdims=True)
    e = np.exp(v - m)
    return e / e.sum(axis=-1, keepdims=True)


# --------------------------------------------------------------------------------------------------
# PlanarLayer  (src/bijectors/planar_layer.jl)
# --------------------------------------------------------------------------------------------------


def get_u_hat(u, w):
    """src/bijectors/planar_layer.jl:65-70 -> (u_hat, wT_u_hat)."""
    dt = w.dtype
    wT_u = dt.type(np.dot(w, u))
    u_hat = u + ((log1pexp(-wT_u) - dt.type(1)) / dt.type(np.sum(w * w))) * w
    wT_u_hat = log1pexp(wT_u) - dt.type(1)
    return u_hat.astype(dt), dt.type(wT_u_hat)


def planar_forward(w, u, b, z):
    """with_logabsdet_jacobian(::PlanarLayer, z) -- src/bijectors/planar_layer.jl:73-80,102-110.

    ``z`` is (D,) or (D, N); returns (y, logjac) with logjac scalar or (N,).
    """
    dt = z.dtype
    b = dt.type(np.asarray(b).reshape(-1)[0])  # first(flow.b), :75
    u_hat, wT_u_hat = get_u_hat(u.astype(dt), w.astype(dt))
    wT_z = w.astype(dt) @ z  # aT_b, src/utils.jl:2-4
    a = wT_z + b
    if z.ndim == 1:
        y = z + u_hat * np.tanh(a)
    else:
        y = z + u_hat[:, None] * np.tanh(a)[None, :]  # :78
    with np.errstate(over="ignore"):
        sech2 = (dt.type(1) / np.cosh(a)) ** 2  # abs2(sech(.)), :107
    logjac = np.log1p(wT_u_hat * sech2)
    return y.astype(dt), np.asarray(logjac, dtype=dt)[()]


def find_alpha_partials(alpha, wt_u_hat, b):
    """Partials (∂α/∂wt_y, ∂α/∂wt_u_hat, ∂α/∂b) of find_alpha by the implicit-function theorem --
    ext/BijectorsChainRulesCoreExt.jl:42-46: x = inv(1 + wt_u_hat·sech(α+b)²) -> (x, −tanh(α+b)·x, x − 1)."""
    x = 1.0 / (1.0 + wt_u_hat / np.cosh(alpha + b) ** 2)
    return x, -np.tanh(alpha + b) * x, x - 1.0


def planar_chain_vjp(params, x, ybar, ljbar, b_terms=None):
    """Vector-Jacobian product of a ∘-chain of PlanarLayers (forward direction) -- what reverse-mode AD of
    with_logabsdet_jacobian (src/bijectors/planar_layer.jl:73-80,102-110 through get_u_hat :65-70) yields; the
    reference trains flows this way (docs/src/flows.md:93-100).

    params: list of (w, u, b); x (D, N); ybar (D, N) cotangent of the transformed batch; ljbar (N,) cotangent of the
    accumulated logjac.  Returns (xbar (D, N), [(wbar, ubar, bbar), ...]).  Written layer by layer with stored
    activations (the plain restatement); the device kernels use the algebraically equal reorganisation described
    in DESIGN.md.  A list ``b_terms`` receives, per layer, the N column terms whose sum is b̄."""
    dt = x.dtype
    zs, cache = [x], []
    for (w, u, b) in params:
        w, u = w.astype(dt), u.astype(dt)
        bb = dt.type(np.asarray(b).reshape(-1)[0])
        u_hat, c = get_u_hat(u, w)
        a = w @ zs[-1] + bb
        t = np.tanh(a)
        with np.errstate(over="ignore"):
            s2 = (dt.type(1) / np.cosh(a)) ** 2
        zs.append(zs[-1] + u_hat[:, None] * t[None, :])
        cache.append((w, u, u_hat, c, t, s2))
    yb = ybar.astype(dt).copy()
    grads = [None] * len(params)
    for l in range(len(params) - 1, -1, -1):
        w, u, u_hat, c, t, s2 = cache[l]
        z = zs[l]
        den = dt.type(1) + c * s2
        d = u_hat @ yb                                   # cotangent of tanh(a)
        g = s2 * d + ljbar * (-2 * c * t * s2 / den)     # cotangent of a = wᵀz + b
        uhat_bar = yb @ t                                # Σ_n t_n ȳ_n
        c_bar = np.sum(ljbar * s2 / den)                 # ∂ log1p(c·s2)/∂c
        w_bar = z @ g                                    # direct dependence a = wᵀz + b
        b_bar = np.sum(g)
        if b_terms is not None:
            b_terms.insert(0, g)
        yb = yb + w[:, None] * g[None, :]
        # through get_u_hat: û = u + k(s, q)·w, k = (log1pexp(−s) − 1)/q, s = wᵀu, q = wᵀw; c = log1pexp(s) − 1
        s_ = dt.type(np.dot(w, u))
        q_ = dt.type(np.sum(w * w))
        sig = lambda v: dt.type(1) / (dt.type(1) + np.exp(-v))
        k = (log1pexp(-s_) - dt.type(1)) / q_
        dk_ds = -sig(-s_) / q_
        dk_dq = -k / q_
        uw = dt.type(np.dot(uhat_bar, w))
        u_bar = uhat_bar + (uw * dk_ds + c_bar * sig(s_)) * w
        w_bar = w_bar + k * uhat_bar + uw * (dk_ds * u + dk_dq * 2 * w) + c_bar * sig(s_) * u
        grads[l] = (w_bar.astype(dt), u_bar.astype(dt), dt.type(b_bar))
    return yb.astype(dt), grads


def _get_u_hat_pullback(w, u, uhat_bar, c_bar, dt):
    """Cotangents (w̄, ū) contributed through get_u_hat (planar_layer.jl:65-70): û = u + k(s, q)·w,
    k = (log1pexp(−s) − 1)/q, s = wᵀu, q = wᵀw; c = wᵀû = log1pexp(s) − 1."""
    s_ = dt.type(np.dot(w, u))
    q_ = dt.type(np.sum(w * w))
    sig = lambda v: dt.type(1) / (dt.type(1) + np.exp(-v))
    k = (log1pexp(-s_) - dt.type(1)) / q_
    dk_ds = -sig(-s_) / q_
    dk_dq = -k / q_
    uw = dt.type(np.dot(uhat_bar, w))
    u_bar = uhat_bar + (uw * dk_ds + c_bar * sig(s_)) * w
    w_bar = k * uhat_bar + uw * (dk_ds * u + dk_dq * 2 * w) + c_bar * sig(s_) * u
    return w_bar, u_bar


def planar_inverse_chain_vjp(params, y, xbar, ljbar, b_terms=None):
    """Vector-Jacobian product of with_logabsdet_jacobian(inverse(f_L ∘ … ∘ f_1), y) -- the computation under
    ``logpdf(transformed(d, flow), y)`` that the reference's training example differentiates
    (docs/src/flows.md:66-100).  Inverse layers are applied in the order L, L−1, …, 1 (planar_layer.jl:112-127); α comes
    from find_alpha and is differentiated with the reference's implicit-function rule
    (ext/BijectorsChainRulesCoreExt.jl:42-46, restated in find_alpha_partials).

    params: [(w, u, b)] in FORWARD order; y (D, N); xbar (D, N) cotangent of the recovered x; ljbar (N,) cotangent of the
    accumulated (inverse) logjac.  Returns (ybar, [(wbar, ubar, bbar), ...]) in forward order.  A list ``b_terms``
    receives, per layer in forward order, the N column terms whose sum is b̄."""
    dt = y.dtype
    L = len(params)
    us, cache = [y], []
    for l in range(L - 1, -1, -1):
        w, u = params[l][0].astype(dt), params[l][1].astype(dt)
        bb = dt.type(np.asarray(params[l][2]).reshape(-1)[0])
        u_hat, c = get_u_hat(u, w)
        t_in = w @ us[-1]
        alpha = find_alpha(t_in, c, bb).astype(dt)
        a = alpha + bb
        th = np.tanh(a)
        with np.errstate(over="ignore"):
            s2 = (dt.type(1) / np.cosh(a)) ** 2
        us.append(us[-1] - u_hat[:, None] * th[None, :])   # planar_layer.jl:124
        cache.append((l, w, u, u_hat, c, bb, alpha, th, s2))
    zb = xbar.astype(dt).copy()
    grads = [None] * L
    for k in range(L - 1, -1, -1):          # reverse over the applied inverse layers
        l, w, u, u_hat, c, bb, alpha, th, s2 = cache[k]
        inp = us[k]
        pt, pc, pb = find_alpha_partials(alpha, c, bb)      # ∂α/∂(wᵀy), ∂α/∂c, ∂α/∂b
        X = pt
        th_bar = -(u_hat @ zb)
        uhat_bar = -(zb @ th)
        # logjac of the inverse layer: −log1p(c·sech²(α+b))  (interface.jl:276-281)
        a_bar = s2 * th_bar + ljbar * (2 * c * th * s2 * X)
        c_bar_direct = np.sum(ljbar * (-s2 * X))
        t_bar = a_bar * pt
        c_bar = np.sum(a_bar * pc) + c_bar_direct
        b_bar = np.sum(a_bar * (1 + pb))                    # a = α + b: direct + through α
        if b_terms is not None:
            b_terms.append(a_bar * (1 + pb))  # k = L−1 … 0 runs over l = 0 … L−1
        w_bar = inp @ t_bar
        zb = zb + w[:, None] * t_bar[None, :]
        gw, gu = _get_u_hat_pullback(w, u, uhat_bar, c_bar, dt)
        grads[l] = ((w_bar + gw).astype(dt), gu.astype(dt), dt.type(b_bar))
    return zb.astype(dt), grads


def find_alpha(wt_y, wt_u_hat, b):
    """src/bijectors/planar_layer.jl:160-185, vectorised over ``wt_y``.

    Roots.A42 narrows the bracket to adjacent floats; here: Newton steps safeguarded by bisection on the
    monotone f(a) = a + c*tanh(a+b) - t until the bracket is adjacent floats or f == 0.
    """
    t = np.asarray(wt_y)
    dt = np.result_type(t.dtype, np.asarray(wt_u_hat).dtype, np.asarray(b).dtype)  # promote(...), :162
    if dt.kind != "f":
        dt = np.dtype(np.float64)
    t = np.atleast_1d(t.astype(dt))
    c = dt.type(wt_u_hat)
    bb = dt.type(b)
    delta = dt.type(2) * abs(c)  # :166
    lo = t - delta
    hi = t + delta
    alpha = t.copy()
    active = lo != hi  # empty bracket -> return lower, :171-173
    alpha[~active] = lo[~active]

    def f(a):
        return a + c * np.tanh(a + bb) - t

    flo = f(lo)
    fhi = f(hi)
    # exact roots at the ends
    hit_lo = active & (flo == 0)
    alpha[hit_lo] = lo[hit_lo]
    active &= ~hit_lo
    hit_hi = active & (fhi == 0)
    alpha[hit_hi] = hi[hit_hi]
    active &= ~hit_hi
    x = np.where(active, (lo + hi) / dt.type(2), alpha)
    for _ in range(200):
        if not active.any():
            break
        fx = f(x)
        root = active & (fx == 0)
        alpha[root] = x[root]
        active &= ~root
        neg = fx < 0
        lo = np.where(active & neg, x, lo)
        hi = np.where(active & ~neg, x, hi)
        # converged when lo and hi are adjacent floats
        adj = active & (np.nextafter(lo, hi) >= hi)
        if adj.any():
            # pick the end with the smaller residual
            fl = np.abs(f(lo))
            fh = np.abs(f(hi))
            alpha[adj] = np.where(fl <= fh, lo, hi)[adj]
            active &= ~adj
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            sech2 = (dt.type(1) / np.cosh(x + bb)) ** 2
            newton = x - fx / (dt.type(1) + c * sech2)
        mid = lo + (hi - lo) / dt.type(2)
        ok = np.isfinite(newton) & (newton > lo) & (newton < hi)
        x = np.where(active, np.where(ok, newton, mid), x)
        # guard against Newton stalling on one side: force bisection every few steps
        if _ % 3 == 2:
            x = np.where(active, mid, x)
    alpha[active] = x[active]
    return alpha if np.ndim(wt_y) else alpha[0]


def planar_inverse(w, u, b, y):
    """with_logabsdet_jacobian(Inverse(PlanarLayer), y):
    transform src/bijectors/planar_layer.jl:112-127 + default inverse logjac src/interface.jl:276-281
    (the forward pass is recomputed on the recovered z, as the reference does)."""
    dt = y.dtype
    w = w.astype(dt)
    bb = dt.type(np.asarray(b).reshape(-1)[0])
    u_hat, wT_u_hat = get_u_hat(u.astype(dt), w)
    wT_y = w @ y
    alpha = find_alpha(wT_y, wT_u_hat, bb)
    th = np.tanh(alpha + bb)
    if y.ndim == 1:
        z = y - u_hat * th
    else:
        z = y - u_hat[:, None] * np.asarray(th)[None, :]
    z = z.astype(dt)
    _, lj = planar_forward(w, u, b, z)
    return z, -lj


# --------------------------------------------------------------------------------------------------
# RadialLayer  (src/bijectors/radial_layer.jl)
# --------------------------------------------------------------------------------------------------


def radial_forward(alpha_raw, beta, z0, z):
    """with_logabsdet_jacobian(::RadialLayer, z) -- src/bijectors/radial_layer.jl:43-53,58-72."""
    dt = z.dtype
    a_ = dt.type(np.asarray(alpha_raw).reshape(-1)[0])  # first(.), :41
    be = dt.type(np.asarray(beta).reshape(-1)[0])
    z0 = z0.astype(dt)
    alpha = dt.type(log1pexp(a_))  # :44
    beta_hat = dt.type(-alpha + log1pexp(be))  # :45
    if z.ndim == 1:
        diff = z - z0
        # LinearAlgebra.norm, :47 (scaled 2-norm; equals sqrt(sum(abs2)) up to rounding)
        r = dt.type(np.sqrt(np.sum(diff * diff)))
        y = z + beta_hat / (alpha + r) * diff  # :51
    else:
        diff = z - z0[:, None]
        r = np.sqrt(np.sum(diff * diff, axis=0)).astype(dt)  # :49
        y = z + (beta_hat / (alpha + r))[None, :] * diff
    d = z0.shape[0]
    h_ = dt.type(1) / (alpha + r)  # h(α, r), :36
    logjac = dt.type(d - 1) * np.log(dt.type(1) + beta_hat * h_) + np.log(
        dt.type(1) + beta_hat * h_ + beta_hat * (-(h_ ** 2)) * r
    )  # :68-70
    return y.astype(dt), np.asarray(logjac, dtype=dt)[()]


def radial_chain_vjp(params, x, ybar, ljbar):
    """Vector-Jacobian product of with_logabsdet_jacobian through a ∘-chain of RadialLayers, forward direction
    (src/bijectors/radial_layer.jl:43-53,58-72) -- what reverse-mode AD of the reference computes.

    params: [(alpha_raw, beta, z0)]; x, ybar (D, N); ljbar (N,).  Returns (xbar, [(alpha_raw_bar, beta_bar, z0_bar)]).
    With δ = z − z0, r = ‖δ‖, h = 1/(α+r), s = β̂h, q = β̂ r h²:  y = z + sδ,
    logjac = (D−1)·log(1+s) + log(1+s−q)."""
    dt = x.dtype
    D = x.shape[0]
    zs, cache = [x], []
    for (a_raw, be, z0) in params:
        a_ = dt.type(np.asarray(a_raw).reshape(-1)[0])
        b_ = dt.type(np.asarray(be).reshape(-1)[0])
        z0 = z0.astype(dt)
        alpha = dt.type(log1pexp(a_))
        beta_hat = dt.type(-alpha + log1pexp(b_))
        delta = zs[-1] - z0[:, None]
        r = np.sqrt(np.sum(delta * delta, axis=0))
        h = 1.0 / (alpha + r)
        s = beta_hat * h
        zs.append(zs[-1] + s[None, :] * delta)
        cache.append((a_, b_, z0, alpha, beta_hat, delta, r, h, s))
    yb = ybar.astype(dt).copy()
    grads = [None] * len(params)
    sig = lambda v: dt.type(1) / (dt.type(1) + np.exp(-v))
    for l in range(len(params) - 1, -1, -1):
        a_, b_, z0, alpha, beta_hat, delta, r, h, s = cache[l]
        q = beta_hat * r * h * h
        s_tot = np.sum(delta * yb, axis=0) + ljbar * ((D - 1) / (1 + s) + 1 / (1 + s - q))
        q_bar = -ljbar / (1 + s - q)
        bh_bar = s_tot * h + q_bar * r * h * h
        h_bar = s_tot * beta_hat + q_bar * 2 * beta_hat * r * h
        r_bar = q_bar * beta_hat * h * h - h_bar * h * h
        alpha_bar = -h_bar * h * h
        with np.errstate(divide="ignore", invalid="ignore"):
            kappa = np.where(r > 0, r_bar / r, 0.0)
        z0_bar = -(yb @ s + delta @ kappa)
        yb = yb * (1 + s)[None, :] + delta * kappa[None, :]
        bh = np.sum(bh_bar)
        al = np.sum(alpha_bar) - bh          # β̂ = log1pexp(β) − α
        grads[l] = (dt.type(al * sig(a_)), dt.type(bh * sig(b_)), z0_bar.astype(dt))
    return yb.astype(dt), grads


def radial_chain_vjp_dir(params, inverse_flags, x, ybar, ljbar):
    """radial_chain_vjp for a chain whose layers are applied in EITHER direction (inverse_flags[l] true = Inverse(layer l),
    radial_layer.jl:88-102,124-129): the VJP a reference AD computes through inverse(flow) -- the logpdf / NLL path of a
    radial flow -- or through mixed chains.  Application order = params order.  Returns (xbar, [(α_bar, β_bar, z0_bar)]).

    Inverse layer, input y: δy = y − z0, γ = ‖δy‖, r = root of r² + (A−γ)r − αγ (A = α+β̂, compute_r :124-129),
    ρ = (α+r)/(A+r), z = z0 + ρ δy, lj = −F(r), F = (D−1)·log(1+s) + log(1+s−q), s = β̂h, q = β̂ r h², h = 1/(α+r).
    r is differentiated implicitly: m = 2r + A − γ, ∂r/∂γ = (α+r)/m, ∂r/∂α = γ/m, ∂r/∂A = −r/m."""
    dt = x.dtype
    D = x.shape[0]
    zs, cache = [x], []
    for (a_raw, be, z0), inv in zip(params, inverse_flags):
        a_ = dt.type(np.asarray(a_raw).reshape(-1)[0])
        b_ = dt.type(np.asarray(be).reshape(-1)[0])
        z0 = z0.astype(dt)
        alpha = dt.type(log1pexp(a_))
        A = dt.type(log1pexp(b_))
        beta_hat = dt.type(A - alpha)
        delta = zs[-1] - z0[:, None]
        nrm = np.sqrt(np.sum(delta * delta, axis=0))
        if not inv:
            r = nrm
            s = beta_hat / (alpha + r)
            zs.append(zs[-1] + s[None, :] * delta)
        else:
            a = A - nrm
            r = 0.5 * (np.sqrt(a * a + 4 * alpha * nrm) - a)
            rho = (alpha + r) / (A + r)
            zs.append(z0[:, None] + rho[None, :] * delta)
        cache.append((a_, b_, z0, alpha, beta_hat, A, delta, nrm, r, bool(inv)))
    yb = ybar.astype(dt).copy()
    grads = [None] * len(params)
    sig = lambda v: dt.type(1) / (dt.type(1) + np.exp(-v))
    for l in range(len(params) - 1, -1, -1):
        a_, b_, z0, alpha, beta_hat, A, delta, nrm, r, inv = cache[l]
        h = 1.0 / (alpha + r)
        s = beta_hat * h
        q = beta_hat * r * h * h
        Fs = (D - 1) / (1 + s) + 1 / (1 + s - q)
        Fq = -1 / (1 + s - q)
        if not inv:
            s_tot = np.sum(delta * yb, axis=0) + ljbar * Fs
            q_bar = ljbar * Fq
            bh_bar = s_tot * h + q_bar * r * h * h
            h_bar = s_tot * beta_hat + q_bar * 2 * beta_hat * r * h
            r_bar = q_bar * beta_hat * h * h - h_bar * h * h
            alpha_bar = -h_bar * h * h
            with np.errstate(divide="ignore", invalid="ignore"):
                kappa = np.where(r > 0, r_bar / r, 0.0)
            z0_bar = -(yb @ s + delta @ kappa)
            yb = yb * (1 + s)[None, :] + delta * kappa[None, :]
        else:
            rho = (alpha + r) / (A + r)
            rho_bar = np.sum(delta * yb, axis=0)
            F_bar = -ljbar
            dF_dr = Fs * (-beta_hat * h * h) + Fq * (beta_hat * h * h - 2 * beta_hat * r * h ** 3)
            dF_da = Fs * (-beta_hat * h * h) + Fq * (-2 * beta_hat * r * h ** 3)
            dF_db = Fs * h + Fq * (r * h * h)
            r_bar = rho_bar * beta_hat / (A + r) ** 2 + F_bar * dF_dr
            m = 2 * r + A - nrm
            A_bar = rho_bar * (-(alpha + r) / (A + r) ** 2) + r_bar * (-r / m)
            alpha_bar = rho_bar / (A + r) + F_bar * dF_da + r_bar * nrm / m + A_bar      # dA/dα = 1 at fixed β̂
            bh_bar = F_bar * dF_db + A_bar                                                  # dA/dβ̂ = 1 at fixed α
            gam_bar = r_bar * (alpha + r) / m
            with np.errstate(divide="ignore", invalid="ignore"):
                kappa = np.where(nrm > 0, gam_bar / nrm, 0.0)
            dy_bar = yb * rho[None, :] + delta * kappa[None, :]
            z0_bar = (yb - dy_bar).sum(axis=1)
            yb = dy_bar
        bh = np.sum(bh_bar)
        al = np.sum(alpha_bar) - bh          # β̂ = log1pexp(β) − α
        grads[l] = (dt.type(al * sig(a_)), dt.type(bh * sig(b_)), z0_bar.astype(dt))
    return yb.astype(dt), grads


def compute_r(y_minus_z0, alpha, alpha_plus_beta_hat):
    """src/bijectors/radial_layer.jl:124-129 (vector or per-column for a matrix)."""
    dt = y_minus_z0.dtype
    gamma = np.sqrt(np.sum(y_minus_z0 * y_minus_z0, axis=0)).astype(dt)  # norm, :125
    a = alpha_plus_beta_hat - gamma
    r = (np.sqrt(a * a + dt.type(4) * alpha * gamma) - a) / dt.type(2)
    return r.astype(dt) if np.ndim(r) else dt.type(r)


def radial_inverse(alpha_raw, beta, z0, y):
    """with_logabsdet_jacobian(Inverse(RadialLayer), y):
    src/bijectors/radial_layer.jl:74-86 (vector), :88-102 (matrix) + src/interface.jl:276-281."""
    dt = y.dtype
    a_ = dt.type(np.asarray(alpha_raw).reshape(-1)[0])
    be = dt.type(np.asarray(beta).reshape(-1)[0])
    z0 = z0.astype(dt)
    alpha = dt.type(log1pexp(a_))
    apb = dt.type(log1pexp(be))
    ymz = y - (z0 if y.ndim == 1 else z0[:, None])
    r = compute_r(ymz, alpha, apb)
    gamma = (alpha + r) / (apb + r)
    if y.ndim == 1:
        z = z0 + gamma * ymz
    else:
        z = z0[:, None] + np.asarray(gamma)[None, :] * ymz
    z = z.astype(dt)
    _, lj = radial_forward(alpha_raw, beta, z0, z)
    return z, -lj


# --------------------------------------------------------------------------------------------------
# RationalQuadraticSpline  (src/bijectors/rational_quadratic_spline.jl)
# --------------------------------------------------------------------------------------------------


def rqs_params(raw_widths, raw_heights, raw_derivs, B):
    """Parameter-normalising constructors, src/bijectors/rational_quadratic_spline.jl:99-107 (vector)
    and :109-123 (matrix).  Returns processed (widths, heights, derivatives) with K+1 knots per row."""
    rw = np.asarray(raw_widths)
    dt = rw.dtype
    rh = np.asarray(raw_heights).astype(dt)
    rd = np.asarray(raw_derivs).astype(dt)
    vec = rw.ndim == 1
    if vec:
        rw, rh, rd = rw[None, :], rh[None, :], rd[None, :]
    d = rw.shape[0]
    ws = np.concatenate([np.zeros((d, 1), dt), softmax_rows(rw).astype(dt)], axis=1)
    hs = np.concatenate([np.zeros((d, 1), dt), softmax_rows(rh).astype(dt)], axis=1)
    ds = np.concatenate([np.ones((d, 1), dt), log1pexp(rd).astype(dt), np.ones((d, 1), dt)], axis=1)
    twoB = dt.type(2 * B)
    Bt = dt.type(B)
    W = (twoB * np.cumsum(ws, axis=1, dtype=dt) - Bt).astype(dt)
    H = (twoB * np.cumsum(hs, axis=1, dtype=dt) - Bt).astype(dt)
    if vec:
        return W[0], H[0], ds[0]
    return W, H, ds


def rqs_validate(widths, heights, derivs):
    """Struct asserts, src/bijectors/rational_quadratic_spline.jl:84-85,93-94."""
    if widths.ndim == 1:
        assert len(widths) == len(heights) == len(derivs)
    else:
        assert widths.shape[1] == heights.shape[1] == derivs.shape[1]
    assert np.all(derivs > 0), "derivatives need to be positive"


def _searchsortedfirst(knots, x):
    """Julia searchsortedfirst(knots, x): 1-based index of the first knot >= x (len+1 if none)."""
    return int(np.searchsorted(knots, x, side="left")) + 1


def rqs_forward_scalar(widths, heights, derivs, x):
    """rqs_forward, src/bijectors/rational_quadratic_spline.jl:317-357 (1-based indexing kept)."""
    dt = np.result_type(widths.dtype, np.asarray(x).dtype)
    one = dt.type(1)
    x = dt.type(x)
    W = lambda k: widths[k - 1]  # noqa: E731  (1-based access)
    H = lambda k: heights[k - 1]  # noqa: E731
    Dv = lambda k: derivs[k - 1]  # noqa: E731
    Kn = len(widths)
    if (x <= -W(Kn)) or (x >= W(Kn)):  # :322-324
        return x, dt.type(0) * x
    k = _searchsortedfirst(widths, x) - 1  # :328
    w_k = -W(Kn) if k == 0 else W(k)  # :331
    w = W(k + 1) - w_k
    h_k = -H(Kn) if k == 0 else H(k)  # :335
    dy = H(k + 1) - h_k
    s = dy / w  # :339
    xi = (x - w_k) / w
    d_k = one if k == 0 else Dv(k)  # :342
    d_k1 = one if k == Kn - 1 else Dv(k + 1)
    den = s + (d_k1 + d_k - 2 * s) * xi * (one - xi)  # :346
    num_jl = s ** 2 * (d_k1 * xi ** 2 + 2 * s * xi * (one - xi) + d_k * (one - xi) ** 2)  # :349
    logjac = np.log(num_jl) - 2 * np.log(den)
    num_y = dy * (s * xi ** 2 + d_k * xi * (one - xi))  # :353
    y = h_k + num_y / den
    return dt.type(y), dt.type(logjac)


def rqs_inverse_scalar(widths, heights, derivs, y):
    """rqs_univariate_inverse, src/bijectors/rational_quadratic_spline.jl:183-220."""
    dt = np.result_type(widths.dtype, np.asarray(y).dtype)
    one = dt.type(1)
    y = dt.type(y)
    W = lambda k: widths[k - 1]  # noqa: E731
    H = lambda k: heights[k - 1]  # noqa: E731
    Dv = lambda k: derivs[k - 1]  # noqa: E731
    Kn = len(widths)
    if (y <= -H(Kn)) or (y >= H(Kn)):  # :186-188
        return y
    k = _searchsortedfirst(heights, y) - 1  # :191
    w_k = -W(Kn) if k == 0 else W(k)
    w = W(k + 1) - w_k
    h_k = -H(Kn) if k == 0 else H(k)
    dy = H(k + 1) - h_k
    s = dy / w
    d_k = one if k == 0 else Dv(k)
    d_k1 = one if k == Kn - 1 else Dv(k + 1)
    ds = d_k1 + d_k - 2 * s  # :205
    a1 = dy * (s - d_k) + (y - h_k) * ds  # :208
    a2 = dy * d_k - (y - h_k) * ds  # :210
    a3 = -s * (y - h_k)  # :212
    num = -2 * a3
    den = a2 + np.sqrt(a2 ** 2 - 4 * a1 * a3)  # :216
    xi = num / den
    return dt.type(xi * w + w_k)


def _rqs_bins(knots, v):
    """Vectorised bin lookup: knots (D, Kn), v (D, N) -> 1-based k = searchsortedfirst - 1, shape (D, N)."""
    # number of knots strictly below v  == searchsortedfirst(knots, v) - 1
    return (knots[:, :, None] < v[:, None, :]).sum(axis=1)


def rqs_forward(widths, heights, derivs, x):
    """Batched map-over-columns of the multivariate RQS (reference defines vectors only:
    transform :173-178, logabsdetjac :304-309, with_logabsdet_jacobian :363-367).
    widths/heights/derivs: (D, Kn); x: (D,) or (D, N) -> (y, logjac[N])."""
    vec = x.ndim == 1
    X = x[:, None] if vec else x
    dt = X.dtype
    W = widths.astype(dt)
    Hh = heights.astype(dt)
    Dv = derivs.astype(dt)
    D, Kn = W.shape
    one = dt.type(1)
    Bw = W[:, -1][:, None]
    outside = (X <= -Bw) | (X >= Bw)
    k = _rqs_bins(W, X)  # 1-based k (0..Kn)
    kc = np.clip(k, 0, Kn - 1)
    rows = np.arange(D)[:, None]

    def g1(A, kk):  # A[k] with 1-based k (k>=1)
        return A[rows, np.clip(kk - 1, 0, Kn - 1)]

    w_k = np.where(kc == 0, -Bw, g1(W, kc))
    w = g1(W, kc + 1) - w_k
    h_k = np.where(kc == 0, -Hh[:, -1][:, None], g1(Hh, kc))
    dy = g1(Hh, kc + 1) - h_k
    with np.errstate(divide="ignore", invalid="ignore"):
        s = dy / w
        xi = (X - w_k) / w
        d_k = np.where(kc == 0, one, g1(Dv, kc))
        d_k1 = np.where(kc == Kn - 1, one, g1(Dv, kc + 1))
        den = s + (d_k1 + d_k - 2 * s) * xi * (one - xi)
        num_jl = s ** 2 * (d_k1 * xi ** 2 + 2 * s * xi * (one - xi) + d_k * (one - xi) ** 2)
        lj = np.log(num_jl) - 2 * np.log(den)
        y = h_k + dy * (s * xi ** 2 + d_k * xi * (one - xi)) / den
    y = np.where(outside, X, y).astype(dt)
    lj = np.where(outside, dt.type(0), lj).astype(dt)
    logjac = lj.sum(axis=0, dtype=dt)
    if vec:
        return y[:, 0], logjac[0]
    return y, logjac


def rqs_inverse(widths, heights, derivs, y):
    """with_logabsdet_jacobian(Inverse(RQS), y): transform :227-233 + src/interface.jl:276-281."""
    vec = y.ndim == 1
    Y = y[:, None] if vec else y
    dt = Y.dtype
    W = widths.astype(dt)
    Hh = heights.astype(dt)
    Dv = derivs.astype(dt)
    D, Kn = W.shape
    one = dt.type(1)
    Bh = Hh[:, -1][:, None]
    outside = (Y <= -Bh) | (Y >= Bh)
    k = _rqs_bins(Hh, Y)
    kc = np.clip(k, 0, Kn - 1)
    rows = np.arange(D)[:, None]

    def g1(A, kk):
        return A[rows, np.clip(kk - 1, 0, Kn - 1)]

    w_k = np.where(kc == 0, -W[:, -1][:, None], g1(W, kc))
    w = g1(W, kc + 1) - w_k
    h_k = np.where(kc == 0, -Bh, g1(Hh, kc))
    dy = g1(Hh, kc + 1) - h_k
    with np.errstate(divide="ignore", invalid="ignore"):
        s = dy / w
        d_k = np.where(kc == 0, one, g1(Dv, kc))
        d_k1 = np.where(kc == Kn - 1, one, g1(Dv, kc + 1))
        ds = d_k1 + d_k - 2 * s
        a1 = dy * (s - d_k) + (Y - h_k) * ds
        a2 = dy * d_k - (Y - h_k) * ds
        a3 = -s * (Y - h_k)
        xi = (-2 * a3) / (a2 + np.sqrt(a2 ** 2 - 4 * a1 * a3))
        x = xi * w + w_k
    x = np.where(outside, Y, x).astype(dt)
    _, lj = rqs_forward(W, Hh, Dv, x)
    if vec:
        return x[:, 0], -lj
    return x, -lj


def rqs_vjp(widths, heights, derivs, x, ybar, ljbar, inverse=False):
    """Vector-Jacobian product of with_logabsdet_jacobian through the RationalQuadraticSpline (mapped over columns) --
    what the reference's reverse-mode AD computes through rational_quadratic_spline.jl:317-357 (forward) / :183-220
    (inverse) -- w.r.t. the input and the PROCESSED knot arrays widths / heights / derivatives (D, Kn).
    x: the layer's input (D, N) (the observed y for inverse=True); ybar (D, N) / ljbar (N,): cotangents of the outputs.
    Returns (xbar, Wbar, Hbar, Dbar).  The reverse sweep goes through
      w = x_{k+1} − x_k, Δ = y_{k+1} − y_k, s = Δ/w, ξ = (x − x_k)/w, o = 1 − ξ, p = ξo, ds = d_{k+1} + d_k − 2s,
      den = s + ds·p, a = sξ² + d_k p, y = y_k + Δ·a/den, b = d_{k+1}ξ² + 2sp + d_k o², lj = 2 log s + log b − 2 log den;
    the inverse uses the inverse-function theorem at the recovered x: with f_x = s²b/den², lj_x = (b_ξ/b − 2den_ξ/den)/w and
    ȳ* = (x̄ − l̄·lj_x)/f_x (lj_inv = −lj_f(x)), the input cotangent is ȳ* and the knot cotangents are the forward sweep's
    with (ȳ, l̄) replaced by (−ȳ*, −l̄).  Elements outside the box pass ȳ through; the box edge itself (a knot that also
    selects the identity branch) is not differentiated."""
    dt = x.dtype
    W, Hh, Dv = widths.astype(dt), heights.astype(dt), derivs.astype(dt)
    D, Kn = W.shape
    N = x.shape[1]
    rows = np.arange(D)[:, None] * np.ones((1, N), int)
    lb = np.zeros(N, dt) if ljbar is None else ljbar.astype(dt)
    lb = lb[None, :] * np.ones((D, 1), dt)
    S = Hh if inverse else W
    Bs = S[:, -1][:, None]
    outside = (x <= -Bs) | (x >= Bs)
    k = np.clip(_rqs_bins(S, x), 0, Kn - 1)
    km1, kk = np.clip(k - 1, 0, Kn - 1), k
    xk = np.where(k == 0, -W[:, -1][:, None], W[rows, km1])
    xk1 = W[rows, kk]
    yk = np.where(k == 0, -Hh[:, -1][:, None], Hh[rows, km1])
    yk1 = Hh[rows, kk]
    dk = np.where(k == 0, dt.type(1), Dv[rows, km1])
    dk1 = np.where(k == Kn - 1, dt.type(1), Dv[rows, kk])
    with np.errstate(divide="ignore", invalid="ignore"):
        w = xk1 - xk
        dyv = yk1 - yk
        s = dyv / w
        if inverse:
            yh = x - yk
            dsv = dk1 + dk - 2 * s
            a1 = dyv * (s - dk) + yh * dsv
            a2 = dyv * dk - yh * dsv
            a3 = -s * yh
            xi = -2 * a3 / (a2 + np.sqrt(a2 * a2 - 4 * a1 * a3))
        else:
            xi = (x - xk) / w
        o = 1 - xi
        p = xi * o
        dsv = dk1 + dk - 2 * s
        den = s + dsv * p
        a = s * xi * xi + dk * p
        num = dyv * a
        b = dk1 * xi * xi + 2 * s * p + dk * o * o
        if inverse:
            f_x = s * s * b / (den * den)
            b_xi = 2 * dk1 * xi + 2 * s * (1 - 2 * xi) - 2 * dk * o
            den_xi = dsv * (1 - 2 * xi)
            lj_x = (b_xi / b - 2 * den_xi / den) / w
            ystar = (ybar.astype(dt) - lb * lj_x) / f_x      # cotangent of the observed y
            yb_, lb_ = -ystar, -lb
        else:
            yb_, lb_ = ybar.astype(dt), lb
        num_b = yb_ / den
        den_b = -yb_ * num / (den * den) - 2 * lb_ / den
        yk_b = yb_.copy()
        b_b = lb_ / b
        s_b = 2 * lb_ / s
        dyv_b = num_b * a
        a_b = num_b * dyv
        s_b = s_b + a_b * xi * xi
        xi_b = a_b * 2 * s * xi
        dk_b = a_b * p
        p_b = a_b * dk
        dk1_b = b_b * xi * xi
        xi_b = xi_b + b_b * 2 * dk1 * xi
        s_b = s_b + b_b * 2 * p
        p_b = p_b + b_b * 2 * s
        dk_b = dk_b + b_b * o * o
        o_b = b_b * 2 * dk * o
        s_b = s_b + den_b
        ds_b = den_b * p
        p_b = p_b + den_b * dsv
        dk1_b = dk1_b + ds_b
        dk_b = dk_b + ds_b
        s_b = s_b - 2 * ds_b
        xi_b = xi_b + p_b * o
        o_b = o_b + p_b * xi
        xi_b = xi_b - o_b
        x_b = xi_b / w
        xk_b = -xi_b / w
        w_b = -xi_b * xi / w
        dyv_b = dyv_b + s_b / w
        w_b = w_b - s_b * s / w
        yk1_b = dyv_b
        yk_b = yk_b - dyv_b
        xk1_b = w_b
        xk_b = xk_b - w_b
    inside = ~outside
    xbar = np.where(outside, ybar.astype(dt), ystar if inverse else x_b).astype(dt)
    Wb, Hb, Db = np.zeros((D, Kn), dt), np.zeros((D, Kn), dt), np.zeros((D, Kn), dt)

    def scatter(T, idx, val, mask):
        np.add.at(T, (rows[mask], idx[mask]), val[mask])

    last = np.full_like(k, Kn - 1)
    m1, m0 = inside & (k >= 1), inside & (k == 0)
    scatter(Wb, km1, xk_b, m1)
    scatter(Wb, last, -xk_b, m0)            # k == 0: x_k = −widths[end]
    scatter(Wb, kk, xk1_b, inside)
    scatter(Hb, km1, yk_b, m1)
    scatter(Hb, last, -yk_b, m0)
    scatter(Hb, kk, yk1_b, inside)
    scatter(Db, km1, dk_b, m1)              # k == 0: d_k = 1 (constant)
    scatter(Db, kk, dk1_b, inside & (k < Kn - 1))  # k == Kn−1: d_{k+1} = 1 (constant)
    return xbar, Wb, Hb, Db


# --------------------------------------------------------------------------------------------------
# PartitionMask / Coupling  (src/bijectors/coupling.jl), Shift / Scale
# --------------------------------------------------------------------------------------------------


@dataclass
class PartitionMask:
    """src/bijectors/coupling.jl:51-118.  Indices are 1-based like the reference; the sparse 0/1
    selector matrices are represented by their index lists (A_i[idx_i[j], j] = 1)."""

    n: int
    indices_1: np.ndarray
    indices_2: np.ndarray
    indices_3: np.ndarray

    @staticmethod
    def make(n, indices_1, indices_2=None, indices_3=None):
        i1 = np.asarray(list(indices_1), dtype=np.int64)
        if indices_2 is None and indices_3 is None:
            # PartitionMask(n, indices): split, :107-115
            i2 = np.asarray([i for i in range(1, n + 1) if i not in set(i1.tolist())], dtype=np.int64)
            i3 = np.zeros((0,), dtype=np.int64)
        elif indices_3 is None:
            i2 = np.asarray(list(indices_2), dtype=np.int64)
            used = set(i1.tolist()) | set(i2.tolist())
            i3 = np.asarray([i for i in range(1, n + 1) if i not in used], dtype=np.int64)  # :85-92
        elif indices_2 is None:
            i3 = np.asarray(list(indices_3), dtype=np.int64)
            used = set(i1.tolist()) | set(i3.tolist())
            i2 = np.asarray([i for i in range(1, n + 1) if i not in used], dtype=np.int64)  # :94-101
        else:
            i2 = np.asarray(list(indices_2), dtype=np.int64)
            i3 = np.asarray(list(indices_3), dtype=np.int64)
        return PartitionMask(n, i1, i2, i3)


def partition(m: PartitionMask, x):
    """src/bijectors/coupling.jl:132-134: (A_1' x, A_2' x, A_3' x)."""
    return x[m.indices_1 - 1], x[m.indices_2 - 1], x[m.indices_3 - 1]


def combine(m: PartitionMask, x_1, x_2, x_3):
    """src/bijectors/coupling.jl:125: A_1 x_1 + A_2 x_2 + A_3 x_3."""
    shape = (m.n,) + tuple(np.shape(x_1)[1:])
    dt = np.result_type(x_1, x_2, x_3) if np.size(x_3) else np.result_type(x_1, x_2)
    out = np.zeros(shape, dtype=dt)
    out[m.indices_1 - 1] += x_1
    out[m.indices_2 - 1] += x_2
    if len(m.indices_3):
        out[m.indices_3 - 1] += x_3
    return out


@dataclass
class Shift:
    """src/bijectors/shift.jl:4-24."""

    a: object

    def wladj(self, x):
        x = np.asarray(x)
        return self.a + x, x.dtype.type(0)  # zero(eltype(x)), :21

    def inv_wladj(self, y):
        y = np.asarray(y)
        return (-np.asarray(self.a)) + y, y.dtype.type(0)  # inverse(b) = Shift(-a), :12


@dataclass
class Scale:
    """src/bijectors/scale.jl:1-39 (scalar / vector ``a``)."""

    a: object

    def _logjac(self, x):
        a = np.asarray(self.a)
        x = np.asarray(x)
        if a.ndim == 0:
            return np.log(np.abs(a)) * (x.size if x.ndim else 1)  # :26-28
        return np.sum(np.log(np.abs(a)))  # :31-32

    def wladj(self, x):
        return np.asarray(self.a) * np.asarray(x), self._logjac(x)

    def inv_wladj(self, y):
        ia = 1.0 / np.asarray(self.a)  # inv.(a), :15-16
        return ia * np.asarray(y), Scale(ia)._logjac(y)


@dataclass
class ComposedLaw:
    """outer ∘ inner for coupling laws (ChangesOfVariables ComposedFunction rule)."""

    outer: object
    inner: object

    def wladj(self, x):
        y1, l1 = self.inner.wladj(x)
        y, l2 = self.outer.wladj(y1)
        return y, l1 + l2

    def inv_wladj(self, y):
        x1, l1 = self.outer.inv_wladj(y)
        x, l2 = self.inner.inv_wladj(x1)
        return x, l1 + l2


def coupling_forward(theta: Callable, mask: PartitionMask, x):
    """with_logabsdet_jacobian(::Coupling, x::vector) -- src/bijectors/coupling.jl:206-215."""
    x_1, x_2, x_3 = partition(mask, x)
    b = theta(x_2)
    y_1, logjac = b.wladj(x_1)
    return combine(mask, y_1, x_2, x_3), logjac


def coupling_inverse(theta: Callable, mask: PartitionMask, y):
    """with_logabsdet_jacobian(::Inverse{<:Coupling}, y) -- src/bijectors/coupling.jl:217-228."""
    y_1, y_2, y_3 = partition(mask, y)
    b = theta(y_2)
    x_1, logjac = b.inv_wladj(y_1)
    return combine(mask, x_1, y_2, y_3), logjac


def affine_law(Wm, c):
    """The affine coupling law θ(x₂) = Shift(t) ∘ Scale(exp.(s)), [s;t] = W·x₂ + c (SURVEY §8 a12):
    Scale src/bijectors/scale.jl:13,31, Shift src/bijectors/shift.jl:14,21."""

    def theta(x_2):
        st = Wm @ x_2 + c
        n1 = st.shape[0] // 2
        return ComposedLaw(Shift(st[n1:]), Scale(np.exp(st[:n1])))

    return theta


def coupling_affine_forward(idx1, idx2, Wm, c, x):
    """Batched (map over columns) affine coupling, SURVEY Appendix A.6.
    idx1/idx2 are 1-based row lists; Wm is (2*n1, n2); x is (D,) or (D, N)."""
    vec = x.ndim == 1
    X = x[:, None] if vec else x
    dt = X.dtype
    i1 = np.asarray(idx1) - 1
    i2 = np.asarray(idx2) - 1
    n1 = len(i1)
    st = Wm.astype(dt) @ X[i2] + c.astype(dt)[:, None]
    s, t = st[:n1], st[n1:]
    Y = X.copy()
    Y[i1] = np.exp(s) * X[i1] + t
    # logjac = Σ log|exp(s_j)|  (scale.jl:31) -- evaluated as Σ s_j (identical unless exp overflows)
    logjac = s.sum(axis=0, dtype=dt)
    if vec:
        return Y[:, 0], logjac[0]
    return Y, logjac


def coupling_affine_inverse(idx1, idx2, Wm, c, y):
    """Inverse affine coupling: x₁ = inv.(exp(s)) .* (y₁ + (-t)) (shift.jl:12, scale.jl:15-16)."""
    vec = y.ndim == 1
    Y = y[:, None] if vec else y
    dt = Y.dtype
    i1 = np.asarray(idx1) - 1
    i2 = np.asarray(idx2) - 1
    n1 = len(i1)
    st = Wm.astype(dt) @ Y[i2] + c.astype(dt)[:, None]
    s, t = st[:n1], st[n1:]
    X = Y.copy()
    X[i1] = (dt.type(1) / np.exp(s)) * (Y[i1] + (-t))
    logjac = -s.sum(axis=0, dtype=dt)
    if vec:
        return X[:, 0], logjac[0]
    return X, logjac


def coupling_affine_vjp(idx1, idx2, Wm, c, x, ybar, ljbar, inverse=False):
    """Vector-Jacobian product of with_logabsdet_jacobian through the affine coupling (what the reference's reverse-mode
    AD computes for coupling.jl:206-228 with the law Shift(t)∘Scale(exp.(s)); `combine`'s pullback,
    ext/BijectorsChainRulesCoreExt.jl:48-62, is the row scatter of the three cotangent blocks).
    x: the layer's INPUT (D, N) (the observed y for inverse=True), ybar (D, N) / ljbar (N,): cotangents of the two outputs.
    Returns (xbar (D, N), Wbar (2n1, n2), cbar (2n1,)), parameter cotangents summed over the columns.
      forward : y1 = e^s x1 + t, lj = Σ s      =>  x̄1 = e^s ȳ1,  s̄ = ȳ1 e^s x1 + l̄,  t̄ = ȳ1
      inverse : x1 = (y1 − t) e^−s, lj = −Σ s  =>  ȳ1 = e^−s x̄1, s̄ = −x1 x̄1 − l̄,   t̄ = −e^−s x̄1
      both    : x̄2 = ȳ2 + Wᵀ[s̄; t̄],  W̄ = [s̄; t̄] x2ᵀ,  c̄ = Σ_n [s̄; t̄],  x̄3 = ȳ3."""
    dt = x.dtype
    i1, i2 = np.asarray(idx1) - 1, np.asarray(idx2) - 1
    n1 = len(i1)
    Wm, c = Wm.astype(dt), c.astype(dt)
    st = Wm @ x[i2] + c[:, None]
    sv, tv = st[:n1], st[n1:]
    lb = np.zeros(x.shape[1], dt) if ljbar is None else ljbar.astype(dt)
    xbar = ybar.astype(dt).copy()
    if not inverse:
        e = np.exp(sv)
        xbar[i1] = e * ybar[i1]
        sbar = ybar[i1] * e * x[i1] + lb[None, :]
        tbar = ybar[i1].astype(dt)
    else:
        em = np.exp(-sv)
        x1 = (x[i1] - tv) * em
        xbar[i1] = em * ybar[i1]
        sbar = -x1 * ybar[i1] - lb[None, :]
        tbar = -em * ybar[i1]
    stbar = np.concatenate([sbar, tbar], axis=0)
    xbar[i2] = ybar[i2] + Wm.T @ stbar
    return xbar, stbar @ x[i2].T, stbar.sum(axis=1)


# --------------------------------------------------------------------------------------------------
# InvertibleBatchNorm  (src/bijectors/normalise.jl)
# --------------------------------------------------------------------------------------------------


@dataclass
class BatchNormParams:
    """InvertibleBatchNorm(chs; eps=1f-5, mtm=1f-1) defaults, src/bijectors/normalise.jl:26-37."""

    b: np.ndarray
    logs: np.ndarray
    m: np.ndarray
    v: np.ndarray
    eps: float = np.float32(1e-5)
    mtm: float = np.float32(1e-1)

    @staticmethod
    def default(chs, dtype=np.float32):
        dt = np.dtype(dtype)
        return BatchNormParams(
            np.zeros(chs, dt), np.zeros(chs, dt), np.zeros(chs, dt), np.ones(chs, dt), dt.type(1e-5), dt.type(1e-1)
        )


def batchnorm_forward(bn: BatchNormParams, x, training=False):
    """src/bijectors/normalise.jl:41-69.  x is (C, N) (channels = ndims-1 axis).  ``training=True``
    follows :51-60 and returns the updated moving stats as a third value."""
    if x.ndim < 2 or x.shape[-2] != len(bn.b):
        raise ValueError(f"InvertibleBatchNorm expected {len(bn.b)} channels, got {x.shape[-2] if x.ndim >= 2 else x.shape}")
    dt = x.dtype
    logs = bn.logs.astype(dt)[:, None]
    s = np.exp(logs)
    b = bn.b.astype(dt)[:, None]
    new_stats = None
    if training:
        n = x.shape[-1]
        m = x.mean(axis=-1, keepdims=True)
        v = ((x - m) ** 2).sum(axis=-1, keepdims=True) / dt.type(n)
        mtm = dt.type(bn.mtm)
        new_m = (1 - mtm) * bn.m + mtm * m[:, 0]
        new_v = (1 - mtm) * bn.v + (mtm * n / (n - 1)) * v[:, 0]
        new_stats = (new_m.astype(bn.m.dtype), new_v.astype(bn.v.dtype))
    else:
        m = bn.m.astype(dt)[:, None]
        v = bn.v.astype(dt)[:, None]
    eps = dt.type(bn.eps)
    result = s * (x - m) / np.sqrt(v + eps) + b  # :66
    lj = np.sum(logs - np.log(v + eps) / dt.type(2), dtype=dt)
    logabsdetjac = np.full(x.shape[-1], lj, dtype=dt)  # fill(...), :67
    if training:
        return result.astype(dt), logabsdetjac, new_stats
    return result.astype(dt), logabsdetjac


def batchnorm_inverse(bn: BatchNormParams, y):
    """src/bijectors/normalise.jl:74-86 (eval mode only, asserted at :75)."""
    dt = y.dtype
    s = np.exp(bn.logs.astype(dt))[:, None]
    b = bn.b.astype(dt)[:, None]
    m = bn.m.astype(dt)[:, None]
    v = bn.v.astype(dt)[:, None]
    x = (y - b) / s * np.sqrt(v + dt.type(bn.eps)) + m  # :84
    x = x.astype(dt)
    _, lj = batchnorm_forward(bn, x)
    return x, -lj


def batchnorm_eval_vjp(bn: BatchNormParams, x, ybar, ljbar, inverse=False):
    """Vector-Jacobian product of the eval-mode InvertibleBatchNorm (normalise.jl:61-67 forward, :74-86 inverse) w.r.t. the
    input and the trainable fields b, logs (Functors.@functor InvertibleBatchNorm (b, logs); m, v are statistics).
      forward : y = A (x − m) + b, A = e^logs / sqrt(v+eps), lj = Σ_c (logs_c − ½ log(v_c+eps))
                x̄ = A ȳ,  b̄ = Σ_n ȳ,  l̄ogs = Σ_n ȳ ⊙ (y − b) + Σ_n l̄
      inverse : x = (y − b)/A + m, lj = −Σ_c(...)
                ȳ = x̄ / A,  b̄ = −Σ_n x̄/A,  l̄ogs = −Σ_n x̄ ⊙ (x − m) − Σ_n l̄
    Returns (input cotangent (C, N), bbar (C,), logsbar (C,))."""
    dt = x.dtype
    A = (np.exp(bn.logs.astype(dt)) / np.sqrt(bn.v.astype(dt) + dt.type(bn.eps)))[:, None]
    b, m = bn.b.astype(dt)[:, None], bn.m.astype(dt)[:, None]
    lsum = dt.type(0) if ljbar is None else ljbar.astype(dt).sum()
    if not inverse:
        y = A * (x - m) + b
        return A * ybar, ybar.sum(axis=1), (ybar * (y - b)).sum(axis=1) + lsum
    xr = (x - b) / A + m
    return ybar / A, -(ybar / A).sum(axis=1), -(ybar * (xr - m)).sum(axis=1) - lsum


# --------------------------------------------------------------------------------------------------
# Permute  (src/bijectors/permute.jl)
# --------------------------------------------------------------------------------------------------


def permute_matrix_from_indices(indices):
    """Permute(indices::Vector{Int}), src/bijectors/permute.jl:90-100: A[idx, i] = 1."""
    n = len(indices)
    A = np.zeros((n, n))
    for i, idx in enumerate(indices, start=1):
        A[idx - 1, i - 1] = 1.0
    return A


def permute_matrix_from_pairs(n, *pairs):
    """Permute(n, src=>dst...) and Permute(n, [srcs]=>[dsts]...), src/bijectors/permute.jl:102-150.
    Raises ValueError where the reference raises ArgumentError (@argcheck)."""
    A = np.eye(n)
    dests, sources = set(), set()
    for src, dst in pairs:
        srcs = list(src) if np.ndim(src) else [src]
        dsts = list(dst) if np.ndim(dst) else [dst]
        if len(srcs) != len(dsts):
            raise ValueError(f"{srcs} => {dsts} is not bijective")  # :132
        for s_, d_ in zip(srcs, dsts):
            if d_ in dests:
                raise ValueError(f"{d_} used more than once")
            if s_ in sources:
                raise ValueError(f"{s_} used more than once")
            dests.add(d_)
            sources.add(s_)
            A[d_ - 1, s_ - 1] = 1.0
            A[s_ - 1, s_ - 1] = 0.0
    if (sources & dests) != (sources | dests):  # :119, :145
        raise ValueError(f"{sources} ∩ {dests} ≠ {sources} ∪ {dests}")
    return A


def permute_dst_of_src(A):
    """Index form of a permutation matrix: y = A x  <=>  y[dst[i]] = x[i] (0-based dst)."""
    A = np.asarray(A)
    if not (np.all((A == 0) | (A == 1)) and np.all(A.sum(0) == 1) and np.all(A.sum(1) == 1)):
        raise ValueError("not a permutation matrix")
    return np.argmax(A, axis=0).astype(np.int64)


def permute_forward(A, x):
    """transform(b::Permute, x) = A * x (src/bijectors/permute.jl:152); logjac zero (:155).
    Implemented as index movement so every payload (NaN, -0.0) is preserved bit-for-bit."""
    dst = permute_dst_of_src(A)
    y = np.empty_like(x)
    y[dst] = x
    lj = np.zeros(x.shape[1], x.dtype) if x.ndim == 2 else x.dtype.type(0)
    return y, lj


def permute_inverse(A, y):
    """inverse(b::Permute) = Permute(transpose(A)), src/bijectors/permute.jl:153."""
    return permute_forward(np.asarray(A).T, y)


# --------------------------------------------------------------------------------------------------
# elementwise exp/log, Stacked  (src/bijectors/exp_log.jl, src/bijectors/stacked.jl)
# --------------------------------------------------------------------------------------------------


def elementwise_exp(x):
    """with_logabsdet_jacobian(elementwise(exp), x) = (exp.(x), sum(x)):
    src/interface.jl:33, src/bijectors/exp_log.jl:6 (+ ChangesOfVariables Fix1{broadcast} rule)."""
    return np.exp(x), np.sum(x, dtype=x.dtype)


def elementwise_log(x):
    """(log.(x), -sum(log, x)) -- src/bijectors/exp_log.jl:9."""
    return np.log(x), -np.sum(np.log(x), dtype=x.dtype)


class EW:
    """Elementwise law codes shared with the device ABI (include/b2b.h, B2B_EW_*)."""

    IDENTITY, EXP, LOG, SHIFT, SCALE, LEAKY_RELU, LOGIT, TRUNCATED = 0, 1, 2, 3, 4, 5, 6, 7


def _logit(z):
    """LogExpFunctions.logit: log(z / (1 - z))."""
    return np.log(z / (1 - z))


def _logistic(y):
    """LogExpFunctions.logistic: 1 / (1 + exp(-y))."""
    return 1 / (1 + np.exp(-y))


def _clamp(x, a, b):
    """_clamp (src/Bijectors.jl:95-100)."""
    return np.where(x < a, a, np.where(x > b, b, x))


def logit_forward(a, b, x):
    """with_logabsdet_jacobian(Logit(a, b), x) per element (src/bijectors/logit.jl:15-29): returns (y, per-element logjac)."""
    dt = x.dtype
    a, b = dt.type(a), dt.type(b)
    return _logit((x - a) / (b - a)), -np.log((x - a) * (b - x) / (b - a))


def logit_inverse(a, b, y):
    """transform(Inverse{Logit}) (logit.jl:19-21) and the default inverse log-Jacobian −logabsdetjac(Logit, x)
    (src/interface.jl:276-281)."""
    dt = y.dtype
    a, b = dt.type(a), dt.type(b)
    x = (b - a) * _logistic(y) + a
    return x, np.log((x - a) * (b - x) / (b - a))


def truncated_forward(lb, ub, x):
    """TruncatedBijector(lb, ub): transform :15-31, logabsdetjac :50-66 (per element, before the sum)."""
    dt = x.dtype
    a, b = dt.type(lb), dt.type(ub)
    xc = _clamp(x, a, b)
    lo, hi = np.isfinite(a), np.isfinite(b)
    if lo and hi:
        return _logit((xc - a) / (b - a)), -np.log((xc - a) * (b - xc) / (b - a))
    if lo:
        return np.log(xc - a), -np.log(xc - a)
    if hi:
        return np.log(b - xc), -np.log(b - xc)
    return xc, np.zeros_like(xc)


def truncated_inverse(lb, ub, y):
    """Inverse{TruncatedBijector}: transform :33-48, logabsdetjac :68-86 (per element)."""
    dt = y.dtype
    a, b = dt.type(lb), dt.type(ub)
    lo, hi = np.isfinite(a), np.isfinite(b)
    if lo and hi:
        ay = np.abs(y)
        return _clamp((b - a) * _logistic(y) + a, a, b), np.log(b - a) - ay - 2 * log1pexp(-ay)
    if lo:
        return _clamp(np.exp(y) + a, a, b), y.copy()
    if hi:
        return _clamp(b - np.exp(y), a, b), y.copy()
    return _clamp(y, a, b), np.zeros_like(y)


def stacked_forward(ops: Sequence[Tuple[int, float]], ranges: Sequence[Tuple[int, int]], x):
    """Stacked(bs, ranges) with elementwise blocks -- src/bijectors/stacked.jl:157-166 (transform),
    :168-193 (logabsdetjac), :242-252 (with_logabsdet_jacobian).  ``ranges`` are 1-based inclusive
    (lo, hi) like Julia UnitRanges; ``ops[i] = (code, a)``.  x is (D,) or (D, N)."""
    length_in = sum(hi - lo + 1 for lo, hi in ranges)
    if length_in != x.shape[0]:
        raise ValueError(f"input length mismatch ({length_in} != {x.shape[0]})")  # :158-160
    dt = x.dtype
    y = np.empty_like(x)
    lj = np.zeros(x.shape[1:], dt)
    for op, (lo, hi) in zip(ops, ranges):
        code, a = op[0], op[1]
        blk = x[lo - 1 : hi]
        nrow = hi - lo + 1
        if code == EW.LOGIT:  # ops entry (code, a, b)
            yb, le = logit_forward(a, op[2], blk)
            l = le.sum(axis=0, dtype=dt)
        elif code == EW.TRUNCATED:
            yb, le = truncated_forward(a, op[2], blk)
            l = le.sum(axis=0, dtype=dt)
        elif code == EW.IDENTITY:
            yb, l = blk, 0
        elif code == EW.EXP:
            yb, l = np.exp(blk), blk.sum(axis=0, dtype=dt)
        elif code == EW.LOG:
            yb, l = np.log(blk), -np.log(blk).sum(axis=0, dtype=dt)
        elif code == EW.SHIFT:
            yb, l = dt.type(a) + blk, 0
        elif code == EW.SCALE:
            yb, l = dt.type(a) * blk, dt.type(np.log(abs(a)) * nrow)
        elif code == EW.LEAKY_RELU:  # src/bijectors/leaky_relu.jl:18-29
            mask = blk < 0
            J = np.where(mask, dt.type(a), dt.type(1))
            yb, l = J * blk, np.log(np.abs(J)).sum(axis=0, dtype=dt)
        else:
            raise ValueError(code)
        y[lo - 1 : hi] = yb
        lj = lj + l
    return y, np.asarray(lj, dtype=dt)[()]


def stacked_inverse(ops, ranges, y):
    if any(op[0] in (EW.LOGIT, EW.TRUNCATED) for op in ops):  # laws whose inverse is not another code of the table
        dt = y.dtype
        x = np.empty_like(y)
        lj = np.zeros(y.shape[1:], dt)
        for op, (lo, hi) in zip(ops, ranges):
            blk = y[lo - 1 : hi]
            if op[0] == EW.LOGIT:
                xb, le = logit_inverse(op[1], op[2], blk)
                l = le.sum(axis=0, dtype=dt)
            elif op[0] == EW.TRUNCATED:
                xb, le = truncated_inverse(op[1], op[2], blk)
                l = le.sum(axis=0, dtype=dt)
            else:
                xb, l = stacked_inverse([op], [(1, hi - lo + 1)], blk)
            x[lo - 1 : hi] = xb
            lj = lj + l
        return x, np.asarray(lj, dtype=dt)[()]
    inv = []
    for op in ops:
        code, a = op[0], op[1]
        if code == EW.EXP:
            inv.append((EW.LOG, a))
        elif code == EW.LOG:
            inv.append((EW.EXP, a))
        elif code == EW.SHIFT:
            inv.append((EW.SHIFT, -a))
        elif code == EW.SCALE:
            inv.append((EW.SCALE, 1.0 / a))
        elif code == EW.LEAKY_RELU:
            inv.append((EW.LEAKY_RELU, 1.0 / a))  # inverse(b) = LeakyReLU(inv(α)), leaky_relu.jl:16
        else:
            inv.append((code, a))
    return stacked_forward(inv, ranges, y)


# --------------------------------------------------------------------------------------------------
# Sampling: Philox4x32-10 + Box-Muller (the device generator of rand(td, n), include/b2b.h)
# --------------------------------------------------------------------------------------------------
# The reference draws base samples with Julia's RNGs (`randn(rng, ...)`, transformed_distribution.jl:212-224), whose
# streams cannot be reproduced here; what is restated is the generator the DEVICE path uses -- Philox4x32-10 of Salmon,
# Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3" (SC'11; Random123, cuRAND) -- pinned by the three
# known-answer vectors of Random123's kat_vectors (tests/test_oracle_golden.py).


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Ten rounds of Philox-4x32 on uint32 arrays (counter words c0..c3, key words k0, k1)."""
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    c0, c1, c2, c3 = (np.asarray(c, np.uint32) for c in (c0, c1, c2, c3))
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = M0 * c0.astype(np.uint64)
        p1 = M1 * c2.astype(np.uint64)
        hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & mask).astype(np.uint32)
        hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & mask).astype(np.uint32)
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint32(k0), lo1, hi0 ^ c3 ^ np.uint32(k1), lo0
        k0 = (k0 + 0x9E3779B9) & 0xFFFFFFFF
        k1 = (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def philox_normals(seed, offset, D, N, column_offset=0, mu=None, sigma=None):
    """The D x N base samples of b2b_randn_f32 / b2b_chain_sample_f32 in float64: rows 4k..4k+3 of global column n come
    from the counter (lo32(n), hi32(n), k, lo32(offset)) under the key (lo32(seed), hi32(seed)); u = x·2^-32 + 2^-33
    evaluated in float32 (as the device does), Box-Muller z0 = sqrt(-2 ln u1)·cos(2π u2), z1 = …·sin(2π u2) in float64."""
    Dc = (D + 3) // 4
    n = np.arange(N, dtype=np.uint64) + np.uint64(column_offset)
    nn, kk = np.meshgrid(n, np.arange(Dc, dtype=np.uint32), indexing="xy")  # (Dc, N)
    o = philox4x32_10((nn & np.uint64(0xFFFFFFFF)).astype(np.uint32), (nn >> np.uint64(32)).astype(np.uint32), kk,
                      np.full(kk.shape, int(offset) & 0xFFFFFFFF, np.uint32), int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF)
    f = np.float32
    u = [(w.astype(f) * f(2.3283064365386963e-10) + f(1.1641532182693481e-10)).astype(np.float64) for w in o]
    z = np.empty((Dc, 4, N))
    for pair in (0, 1):
        r = np.sqrt(-2.0 * np.log(u[2 * pair]))
        z[:, 2 * pair, :] = r * np.cos(2.0 * np.pi * u[2 * pair + 1])
        z[:, 2 * pair + 1, :] = r * np.sin(2.0 * np.pi * u[2 * pair + 1])
    z = z.reshape(Dc * 4, N)[:D]
    if sigma is not None:
        z = z * np.asarray(sigma, np.float64)[:, None]
    if mu is not None:
        z = z + np.asarray(mu, np.float64)[:, None]
    return z


# --------------------------------------------------------------------------------------------------
# MvNormal (Distributions/PDMats), chains, TransformedDistribution
# --------------------------------------------------------------------------------------------------


def mvnormal_diag_logpdf(mu, sigma, x):
    """logpdf(MvNormal(mu, Diagonal(sigma.^2)), x) for x (D,) or (D, N) (Distributions + PDMats):
    -(D*log(2π) + Σ log σ²)/2 - Σ ((x-μ)/σ)² / 2."""
    dt = x.dtype
    D = x.shape[0]
    mu = np.zeros(D, dt) if mu is None else np.asarray(mu, dt)
    sigma = np.ones(D, dt) if sigma is None else np.asarray(sigma, dt)
    zc = (x - (mu if x.ndim == 1 else mu[:, None])) / (sigma if x.ndim == 1 else sigma[:, None])
    const = -(dt.type(D) * dt.type(math.log(2 * math.pi)) + np.sum(np.log(sigma * sigma), dtype=dt)) / dt.type(2)
    return (const - np.sum(zc * zc, axis=0, dtype=dt) / dt.type(2)).astype(dt)[()]


@dataclass
class Layer:
    """One chain element: kind in {planar, radial, rqs, coupling_affine, batchnorm, permute, stacked}."""

    kind: str
    params: dict = field(default_factory=dict)

    def forward(self, x):
        p = self.params
        k = self.kind
        if k == "planar":
            return planar_forward(p["w"], p["u"], p["b"], x)
        if k == "radial":
            return radial_forward(p["alpha_raw"], p["beta"], p["z0"], x)
        if k == "rqs":
            return rqs_forward(p["widths"], p["heights"], p["derivs"], x)
        if k == "coupling_affine":
            return coupling_affine_forward(p["idx1"], p["idx2"], p["W"], p["c"], x)
        if k == "batchnorm":
            if x.ndim == 1:  # the reference needs >= 2 dims; a vector is treated as one column
                y, lj = batchnorm_forward(p["bn"], x[:, None])
                return y[:, 0], lj[0]
            return batchnorm_forward(p["bn"], x)
        if k == "permute":
            return permute_forward(p["A"], x)
        if k == "stacked":
            return stacked_forward(p["ops"], p["ranges"], x)
        raise ValueError(k)

    def inverse(self, y):
        p = self.params
        k = self.kind
        if k == "planar":
            return planar_inverse(p["w"], p["u"], p["b"], y)
        if k == "radial":
            return radial_inverse(p["alpha_raw"], p["beta"], p["z0"], y)
        if k == "rqs":
            return rqs_inverse(p["widths"], p["heights"], p["derivs"], y)
        if k == "coupling_affine":
            return coupling_affine_inverse(p["idx1"], p["idx2"], p["W"], p["c"], y)
        if k == "batchnorm":
            if y.ndim == 1:
                x, lj = batchnorm_inverse(p["bn"], y[:, None])
                return x[:, 0], lj[0]
            return batchnorm_inverse(p["bn"], y)
        if k == "permute":
            return permute_inverse(p["A"], y)
        if k == "stacked":
            return stacked_inverse(p["ops"], p["ranges"], y)
        raise ValueError(k)


def chain_forward(layers: List[Layer], x):
    """with_logabsdet_jacobian(L_n ∘ … ∘ L_1, x): inner-most (layers[0]) first, logjacs added
    (ChangesOfVariables ComposedFunction rule; src/bijectors/composed.jl:4,11-14)."""
    lj = None
    y = x
    for L in layers:
        y, l = L.forward(y)
        lj = l if lj is None else lj + l
    return y, lj


def chain_inverse(layers: List[Layer], y):
    """with_logabsdet_jacobian(inverse(L_n ∘ … ∘ L_1), y): inverse(f∘g) = inverse(g)∘inverse(f)
    (InverseFunctions) -> the last-applied layer is inverted first."""
    lj = None
    x = y
    for L in reversed(layers):
        x, l = L.inverse(x)
        lj = l if lj is None else lj + l
    return x, lj


def transformed_logpdf(layers: List[Layer], mu, sigma, y):
    """logpdf(td::MvTransformed, y::Matrix) -- src/transformed_distribution.jl:165-169."""
    x, lj = chain_inverse(layers, y)
    return mvnormal_diag_logpdf(mu, sigma, x) + lj
