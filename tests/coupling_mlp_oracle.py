"""Reference for the neural-network coupling layer, B2B_COUPLING_MLP: Coupling(θ, mask) (coupling.jl:206-228) with
θ(x₂) = Shift(t) ∘ Scale(exp.(s)), [s; t] = W₂·σ.(W₁·x₂ + c₁) + c₂, σ = tanh or LeakyReLU(a) (v >= 0 ? v : a·v,
leaky_relu.jl:18-29; σ′(0) = 1).

The law is the affine coupling's, so everything after the hidden layer is oracle_np's affine coupling applied to the
stacked column [x₁; h] with h = σ(W₁x₂ + c₁) in the role of x₂: rows 1..n1 are transformed, rows n1+1..n1+H condition,
W = W₂, c = c₂.  Its VJP returns x̄₁, h̄ = W₂ᵀ[s̄; t̄], W̄₂ and c̄₂; the hidden layer's pullback is written here:
v̄ = h̄ ⊙ σ′(v), x̄₂ = ȳ₂ + W₁ᵀv̄, W̄₁ = Σ v̄ x₂ᵀ, c̄₁ = Σ v̄.  ``dtype`` float32 evaluates the same formulas in float32 (the
reference's own float32 error for the parity gates).  idx1 / idx2 are 1-based row lists; W1 is (H, n2), W2 (2·n1, H);
c1 / c2 may be None."""
import numpy as np

from oracle import oracle_np as O


def hidden(W1, c1, x2, act, slope, dtype=np.float64):
    """(h, σ′(v)) for v = W₁x₂ + c₁, x₂ (n2, N)."""
    dt = np.dtype(dtype)
    v = np.asarray(W1, dt) @ np.asarray(x2, dt)
    if c1 is not None:
        v = v + np.asarray(c1, dt)[:, None]
    if act == "tanh":
        h = np.tanh(v)
        return h.astype(dt), (1 - h * h).astype(dt)
    a = dt.type(slope)
    return np.where(v >= 0, v, a * v).astype(dt), np.where(v >= 0, dt.type(1), a).astype(dt)


def _stacked(idx1, idx2, W1, c1, W2, c2, act, slope, x, dt):
    """[x₁; h], the affine coupling's index lists on it, W₂ and c₂ in dt, and σ′(v)."""
    x = np.asarray(x, dt)
    i1, i2 = np.asarray(idx1, int) - 1, np.asarray(idx2, int) - 1
    n1, H = len(i1), np.shape(W1)[0]
    h, dh = hidden(W1, c1, x[i2], act, slope, dt)
    c2 = np.zeros(2 * n1, dt) if c2 is None else np.asarray(c2, dt)
    return np.concatenate([x[i1], h]), np.arange(1, n1 + 1), np.arange(n1 + 1, n1 + H + 1), np.asarray(W2, dt), c2, dh


def _run(affine, idx1, idx2, W1, c1, W2, c2, act, slope, x, dtype):
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    z, j1, j2, W2, c2, _ = _stacked(idx1, idx2, W1, c1, W2, c2, act, slope, x, dt)
    zy, lj = affine(j1, j2, W2, c2, z)
    y = x.copy()
    y[np.asarray(idx1, int) - 1] = zy[: len(j1)]
    return y, np.asarray(lj, dt)


def forward(idx1, idx2, W1, c1, W2, c2, act, slope, x, dtype=np.float64):
    """with_logabsdet_jacobian(Coupling, x) for x (D, N)."""
    return _run(O.coupling_affine_forward, idx1, idx2, W1, c1, W2, c2, act, slope, x, dtype)


def inverse(idx1, idx2, W1, c1, W2, c2, act, slope, y, dtype=np.float64):
    """with_logabsdet_jacobian(Inverse(Coupling), y)."""
    return _run(O.coupling_affine_inverse, idx1, idx2, W1, c1, W2, c2, act, slope, y, dtype)


def vjp(idx1, idx2, W1, c1, W2, c2, act, slope, x, ybar, ljbar, inverse=False, dtype=np.float64):
    """Reverse mode of forward (inverse=False) or inverse (inverse=True) at x (D, N; the observed y for the inverse):
    (x̄ (D, N), dict(W1=(H, n2), c1=(H,), W2=(2n1, H), c2=(2n1,))).  ybar (D, N) / ljbar (N,) may be None (zeros)."""
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    D, N = x.shape
    i1, i2 = np.asarray(idx1, int) - 1, np.asarray(idx2, int) - 1
    n1 = len(i1)
    yb = np.zeros((D, N), dt) if ybar is None else np.asarray(ybar, dt)
    lb = np.zeros(N, dt) if ljbar is None else np.asarray(ljbar, dt)
    z, j1, j2, W2, c2, dh = _stacked(idx1, idx2, W1, c1, W2, c2, act, slope, x, dt)
    zb = np.concatenate([yb[i1], np.zeros_like(dh)])
    zbar, W2b, c2b = O.coupling_affine_vjp(j1, j2, W2, c2, z, zb, lb, inverse=inverse)
    vb = (zbar[n1:] * dh).astype(dt)
    xbar = yb.copy()
    xbar[i1] = zbar[:n1]
    xbar[i2] = yb[i2] + np.asarray(W1, dt).T @ vb
    return xbar, dict(W1=(vb @ x[i2].T).astype(dt), c1=vb.sum(axis=1, dtype=dt), W2=W2b, c2=c2b)


class MLPLayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse (evaluated in the batch's dtype)."""

    kind = "coupling_mlp"

    def __init__(self, idx1, idx2, W1, c1, W2, c2, act="tanh", slope=0.0):
        self.args = (idx1, idx2, W1, c1, W2, c2, act, slope)

    def forward(self, x):
        return forward(*self.args, x, x.dtype)

    def inverse(self, y):
        return inverse(*self.args, y, y.dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        x = np.asarray(x)
        return vjp(*self.args, x, ybar, ljbar, inverse, x.dtype)
