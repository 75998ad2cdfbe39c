"""Reference for the deep neural spline coupling layer, B2B_COUPLING_DEEP_MLP_RQS: Coupling(x₂ ->
RationalQuadraticSpline(…, B), mask) (coupling.jl:206-228) whose raw knots come from an MLP with M >= 2 hidden layers,
h_1 = σ.(W_in·x₂ + c_1), h_l = σ.(W_l·h_{l−1} + c_l) (l = 2..M), v = W_out·h_M + c_out, σ = tanh or LeakyReLU(a).

This composes the existing references: the hidden stack of coupling_deep_mlp_oracle.stack, then spline_coupling_oracle on
the stacked column [x₁; h_M] with h_M in the role of x₂ (W = W_out, c = c_out).  The spline VJP returns x̄₁,
h̄_M = W_outᵀr̄, W̄_out and c̄_out; the pullback through the stack is that of coupling_deep_mlp_oracle: v̄_l = h̄_l ⊙ σ′_l,
h̄_{l−1} = W_lᵀ v̄_l, W̄_l = Σ v̄_l h_{l−1}ᵀ, c̄_l = Σ v̄_l, and x̄₂ = ȳ₂ + h̄_0.  ``dtype`` float32 evaluates the same
formulas in float32 (the reference's own float32 error for the parity gates).  idx1 / idx2 are 1-based row lists;
``weights`` = [W_in (H, n2), W_2 … W_M (H, H), W_out ((3K−1)·n1, H)]; ``biases`` = None or [c_1 … c_M (H),
c_out ((3K−1)·n1)]."""
import numpy as np

import coupling_deep_mlp_oracle as DM
import spline_coupling_oracle as S


def _stacked(idx1, idx2, weights, biases, act, slope, x, dt):
    """[x₁; h_M], the spline coupling's index lists on it, W_out, c_out (None: no biases) and the stack's factors."""
    i1, i2 = np.asarray(idx1, int) - 1, np.asarray(idx2, int) - 1
    n1, H = len(i1), np.shape(weights[0])[0]
    hs, dhs = DM.stack(weights, biases, x[i2], act, slope, dt)
    c_out = None if biases is None else np.asarray(biases[-1], dt)
    z = np.concatenate([x[i1], hs[-1]])
    return z, np.arange(1, n1 + 1), np.arange(n1 + 1, n1 + H + 1), np.asarray(weights[-1], dt), c_out, hs, dhs


def _run(step, idx1, idx2, weights, biases, K, B, act, slope, x, dtype, cols):
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    if cols is not None:
        x = x[:, list(cols)]
    z, j1, j2, W_out, c_out, _, _ = _stacked(idx1, idx2, weights, biases, act, slope, x, dt)
    zy, lj = step(j1, j2, W_out, c_out, K, B, z, dt)
    y = x.copy()
    y[np.asarray(idx1, int) - 1] = zy[: len(j1)]
    return y, np.asarray(lj, dt)


def forward(idx1, idx2, weights, biases, K, B, act, slope, x, dtype=np.float64, cols=None):
    """with_logabsdet_jacobian(Coupling, x) for x (D, N) (or its columns ``cols``)."""
    return _run(S.forward, idx1, idx2, weights, biases, K, B, act, slope, x, dtype, cols)


def inverse(idx1, idx2, weights, biases, K, B, act, slope, y, dtype=np.float64, cols=None):
    """with_logabsdet_jacobian(Inverse(Coupling), y); the network is evaluated on y₂ = x₂."""
    return _run(S.inverse, idx1, idx2, weights, biases, K, B, act, slope, y, dtype, cols)


def vjp(idx1, idx2, weights, biases, K, B, act, slope, x, ybar, ljbar, inverse=False, dtype=np.float64):
    """Reverse mode of forward (inverse=False) or inverse (inverse=True) at x (D, N; the observed y for the inverse):
    (x̄ (D, N), dict(W_in=(H, n2), W_hid=(M−1, H, H), W_out=((3K−1)n1, H), c=(M·H + (3K−1)n1,))).  c̄ is returned
    whether or not the layer has biases.  ybar (D, N) / ljbar (N,) may be None (zeros)."""
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    D, N = x.shape
    i1, i2 = np.asarray(idx1, int) - 1, np.asarray(idx2, int) - 1
    n1 = len(i1)
    yb = np.zeros((D, N), dt) if ybar is None else np.asarray(ybar, dt)
    z, j1, j2, W_out, c_out, hs, dhs = _stacked(idx1, idx2, weights, biases, act, slope, x, dt)
    zb = np.concatenate([yb[i1], np.zeros_like(hs[-1])])
    zbar, W_outb, c_outb = S.vjp(j1, j2, W_out, c_out, K, B, z, zb, ljbar, inverse=inverse, dtype=dt)
    hb = zbar[n1:]
    Wb, cb = [None] * (len(weights) - 1), [None] * (len(weights) - 1)
    for l in range(len(weights) - 2, -1, -1):  # layer l + 1 of the text: h_{l+1} = σ(weights[l]·h_l + c_{l+1})
        vb = (hb * dhs[l]).astype(dt)
        Wb[l] = (vb @ hs[l].T).astype(dt)
        cb[l] = vb.sum(axis=1, dtype=dt)
        hb = np.asarray(weights[l], dt).T @ vb
    xbar = yb.copy()
    xbar[i1] = zbar[:n1]
    xbar[i2] = yb[i2] + hb
    return xbar, dict(W_in=Wb[0], W_hid=np.stack(Wb[1:]), W_out=W_outb, c=np.concatenate(cb + [c_outb]))


class DeepMLPSplineLayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse (evaluated in the batch's dtype).  Its kind is
    the network coupling's: chain_vjp_oracle hands every layer of that kind to the layer's own .vjp, which is what this
    layer needs; nothing else reads the kind."""

    kind = "coupling_mlp"

    def __init__(self, idx1, idx2, weights, biases, K, B, act="tanh", slope=0.0):
        self.args = (idx1, idx2, weights, biases, K, B, act, slope)

    def forward(self, x):
        return forward(*self.args, x, x.dtype)

    def inverse(self, y):
        return inverse(*self.args, y, y.dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        x = np.asarray(x)
        return vjp(*self.args, x, ybar, ljbar, inverse, x.dtype)
