"""Reference for the neural spline coupling layer, B2B_COUPLING_MLP_RQS: Coupling(x₂ -> RationalQuadraticSpline(…, B),
mask) (coupling.jl:206-228) whose raw knots come from a one-hidden-layer network, v = W₂·σ.(W₁·x₂ + c₁) + c₂, σ = tanh
or LeakyReLU(a) (σ′(0) = 1).

The law after the hidden layer is the spline coupling's, so this composes the two existing references: spline_coupling_oracle
on the stacked column [x₁; h] with h = σ(W₁x₂ + c₁) in the role of x₂ (rows 1..n1 transformed, rows n1+1..n1+H
conditioning, W = W₂, c = c₂), and the hidden layer of coupling_mlp_oracle.  The spline VJP returns x̄₁, h̄ = W₂ᵀr̄, W̄₂
and c̄₂; the hidden layer's pullback is v̄ = h̄ ⊙ σ′(v), x̄₂ = ȳ₂ + W₁ᵀv̄, W̄₁ = Σ v̄ x₂ᵀ, c̄₁ = Σ v̄.  ``dtype`` float32
evaluates the same formulas in float32.  idx1 / idx2 are 1-based row lists; W1 is (H, n2), W2 ((3K−1)·n1, H); c1 / c2
may be None."""
import numpy as np

import coupling_mlp_oracle as M
import spline_coupling_oracle as S


def _stacked(idx1, idx2, W1, c1, act, slope, x, dt):
    """[x₁; h], the spline coupling's index lists on it, and σ′(v)."""
    i1, i2 = np.asarray(idx1, int) - 1, np.asarray(idx2, int) - 1
    n1, H = len(i1), np.shape(W1)[0]
    h, dh = M.hidden(W1, c1, x[i2], act, slope, dt)
    return np.concatenate([x[i1], h]), np.arange(1, n1 + 1), np.arange(n1 + 1, n1 + H + 1), dh


def _run(step, idx1, idx2, W1, c1, W2, c2, K, B, act, slope, x, dtype, cols):
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    if cols is not None:
        x = x[:, list(cols)]
    z, j1, j2, _ = _stacked(idx1, idx2, W1, c1, act, slope, x, dt)
    zy, lj = step(j1, j2, W2, c2, K, B, z, dt)
    y = x.copy()
    y[np.asarray(idx1, int) - 1] = zy[: len(j1)]
    return y, np.asarray(lj, dt)


def forward(idx1, idx2, W1, c1, W2, c2, K, B, act, slope, x, dtype=np.float64, cols=None):
    """with_logabsdet_jacobian(Coupling, x) for x (D, N) (or its columns ``cols``)."""
    return _run(S.forward, idx1, idx2, W1, c1, W2, c2, K, B, act, slope, x, dtype, cols)


def inverse(idx1, idx2, W1, c1, W2, c2, K, B, act, slope, y, dtype=np.float64, cols=None):
    """with_logabsdet_jacobian(Inverse(Coupling), y); the network is evaluated on y₂ = x₂."""
    return _run(S.inverse, idx1, idx2, W1, c1, W2, c2, K, B, act, slope, y, dtype, cols)


def vjp(idx1, idx2, W1, c1, W2, c2, K, B, act, slope, x, ybar, ljbar, inverse=False, dtype=np.float64):
    """Reverse mode of forward (inverse=False) or inverse (inverse=True) at x (D, N; the observed y for the inverse):
    (x̄ (D, N), dict(W1=(H, n2), c1=(H,), W2=((3K−1)n1, H), c2=((3K−1)n1,))).  ybar / ljbar may be None (zeros)."""
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    D, N = x.shape
    i1, i2 = np.asarray(idx1, int) - 1, np.asarray(idx2, int) - 1
    n1 = len(i1)
    yb = np.zeros((D, N), dt) if ybar is None else np.asarray(ybar, dt)
    z, j1, j2, dh = _stacked(idx1, idx2, W1, c1, act, slope, x, dt)
    zb = np.concatenate([yb[i1], np.zeros_like(dh)])
    zbar, W2b, c2b = S.vjp(j1, j2, W2, c2, K, B, z, zb, ljbar, inverse=inverse, dtype=dt)
    vb = (zbar[n1:] * dh).astype(dt)
    xbar = yb.copy()
    xbar[i1] = zbar[:n1]
    xbar[i2] = yb[i2] + np.asarray(W1, dt).T @ vb
    return xbar, dict(W1=(vb @ x[i2].T).astype(dt), c1=vb.sum(axis=1, dtype=dt), W2=W2b, c2=c2b)


class MLPSplineLayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse (evaluated in the batch's dtype).  Its kind is
    the network coupling's: chain_vjp_oracle hands every layer of that kind to the layer's own .vjp, which is what this
    layer needs; nothing else reads the kind."""

    kind = "coupling_mlp"

    def __init__(self, idx1, idx2, W1, c1, W2, c2, K, B, act="tanh", slope=0.0):
        self.args = (idx1, idx2, W1, c1, W2, c2, K, B, act, slope)

    def forward(self, x):
        return forward(*self.args, x, x.dtype)

    def inverse(self, y):
        return inverse(*self.args, y, y.dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        x = np.asarray(x)
        return vjp(*self.args, x, ybar, ljbar, inverse, x.dtype)
