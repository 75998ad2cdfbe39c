"""Float64 numpy reference of the masked autoregressive layer, B2B_AUTOREGRESSIVE_MLP (include/b2b.h): MAF / IAF's affine
layer with a one-hidden-layer MADE conditioner.  With 1-based rows r, hidden units k of degree m_k and masks
M₁[k, r] = (r <= m_k), M₂[i, k] = M₂[D+i, k] = (m_k < i):

    u = (M₁⊙W₁) x + c₁,   h = σ.(u),   [s; t] = (M₂⊙W₂) h + c₂,   y = x ⊙ exp.(s) + t,   logjac = Σ s

The inverse recovers x row by row.  Reverse mode follows the rules stated in the layer's documentation: the forward
rule, and for the inverse layer g = v̄ − ℓ̄·∇ᵥΣ s(v), the back substitution Jᵀ w̄ = g, and the forward rule's parameter
sums at v with [s̄; t̄] = −[w̄ ⊙ v ⊙ eˢ + ℓ̄; w̄].  Every function evaluates in `dtype` (float32 gives the reference's own
float32 error for the parity gate).  W1 is (H, D) and W2 (2D, H) in the reference orientation; c1 / c2 may be None."""
import numpy as np


def default_degrees(D, H):
    """MADE's cyclic assignment m_k = ((k−1) mod max(D−1, 1)) + 1."""
    return np.arange(H) % max(D - 1, 1) + 1


def masks(deg, D):
    """(M₁ (H, D), M₂ (2D, H)) as booleans."""
    m = np.asarray(deg, np.int64)
    r = np.arange(1, D + 1)
    M1 = r[None, :] <= m[:, None]
    M2 = np.tile(m[None, :] < r[:, None], (2, 1))
    return M1, M2


def _act(act, slope, u):
    if act == "tanh":
        h = np.tanh(u)
        return h, 1 - h * h
    return np.where(u >= 0, u, slope * u), np.where(u >= 0, 1.0, slope).astype(u.dtype)


class _Net:
    def __init__(self, W1, c1, W2, c2, deg, act, slope, dt):
        W1, W2 = np.asarray(W1, np.float64), np.asarray(W2, np.float64)
        self.H, self.D = W1.shape
        self.M1, self.M2 = masks(deg, self.D)
        self.W1 = np.where(self.M1, W1, 0).astype(dt)  # entries outside the masks are never used (NaN allowed)
        self.W2 = np.where(self.M2, W2, 0).astype(dt)
        self.c1 = np.zeros(self.H, dt) if c1 is None else np.asarray(c1, dt)
        self.c2 = np.zeros(2 * self.D, dt) if c2 is None else np.asarray(c2, dt)
        self.act, self.slope, self.dt = act, dt.type(slope), dt

    def __call__(self, x):
        """u's activation h, σ′(u), s, t at x (D, N)."""
        u = self.W1 @ x + self.c1[:, None]
        h, dh = _act(self.act, self.slope, u)
        st = self.W2 @ h + self.c2[:, None]
        return h.astype(self.dt), dh.astype(self.dt), st[: self.D], st[self.D:]

    def params_vjp(self, x, h, dh, st_bar):
        """(v̄ of the network input, {W1, c1, W2, c2}) for the cotangent [s̄; t̄] of the network output at x."""
        ub = (self.W2.T @ st_bar) * dh
        grads = dict(W1=np.where(self.M1, ub @ x.T, 0), c1=ub.sum(axis=1), W2=np.where(self.M2, st_bar @ h.T, 0),
                     c2=st_bar.sum(axis=1))
        return self.W1.T @ ub, {k: np.asarray(v, self.dt) for k, v in grads.items()}


def forward(W1, c1, W2, c2, deg, act, slope, x, dtype=np.float64):
    """(y, logjac) of the layer at x (D, N)."""
    dt = np.dtype(dtype)
    net = _Net(W1, c1, W2, c2, deg, act, slope, dt)
    x = np.asarray(x, dt)
    _, _, s, t = net(x)
    return (x * np.exp(s) + t).astype(dt), s.sum(axis=0, dtype=dt)


def inverse(W1, c1, W2, c2, deg, act, slope, y, dtype=np.float64):
    """(x, −Σ s(x)) with x recovered row by row: xᵢ = (yᵢ − tᵢ)·exp(−sᵢ), sᵢ and tᵢ from rows 1..i−1."""
    dt = np.dtype(dtype)
    net = _Net(W1, c1, W2, c2, deg, act, slope, dt)
    y = np.asarray(y, dt)
    x = np.zeros_like(y)
    for i in range(net.D):
        _, _, s, t = net(x)  # rows >= i of x are still 0 and do not reach sᵢ, tᵢ
        x[i] = (y[i] - t[i]) / np.exp(s[i])
    _, _, s, _ = net(x)
    return x, -s.sum(axis=0, dtype=dt)


def vjp(W1, c1, W2, c2, deg, act, slope, x, ybar, ljbar, inverse=False, dtype=np.float64):
    """Reverse mode of the layer (inverse=False) or of its inverse (inverse=True) at x (D, N; the observed y for the
    inverse): (x̄, dict(W1 (H, D), c1 (H,), W2 (2D, H), c2 (2D,))), W̄ exactly 0 outside the masks.  c̄ is returned whether
    or not the layer has biases; ybar (D, N) / ljbar (N,) may be None (zeros)."""
    dt = np.dtype(dtype)
    net = _Net(W1, c1, W2, c2, deg, act, slope, dt)
    x = np.asarray(x, dt)
    D, N = x.shape
    yb = np.zeros((D, N), dt) if ybar is None else np.asarray(ybar, dt)
    lb = np.zeros(N, dt) if ljbar is None else np.asarray(ljbar, dt)
    if not inverse:
        h, dh, s, t = net(x)
        e = np.exp(s)
        st_bar = np.concatenate([yb * x * e + lb[None, :], yb])
        xb, grads = net.params_vjp(x, h, dh, st_bar)
        return (yb * e + xb).astype(dt), grads
    v = globals()["inverse"](W1, c1, W2, c2, deg, act, slope, x, dt)[0]
    h, dh, s, t = net(v)
    e = np.exp(s)
    ds = np.concatenate([np.ones((D, N), dt), np.zeros((D, N), dt)])
    g = yb - lb[None, :] * net.params_vjp(v, h, dh, ds)[0]  # v̄ − ℓ̄·∇ᵥΣ s
    wb = np.zeros((D, N), dt)
    for i in range(D - 1, -1, -1):  # Jᵀ w̄ = eˢ ⊙ w̄ + (M₁⊙W₁)ᵀ(σ′ ⊙ (M₂⊙W₂)ᵀ[v ⊙ eˢ ⊙ w̄; w̄]), rows > i known
        a = (net.W2.T @ np.concatenate([v * e * wb, wb])) * dh
        wb[i] = (g[i] - (net.W1.T @ a)[i]) / e[i]
    st_bar = -np.concatenate([wb * v * e + lb[None, :], wb])
    _, grads = net.params_vjp(v, h, dh, st_bar)
    return wb, grads


class AutoregressiveLayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse and of chain_vjp_oracle.chain_vjp (evaluated
    in the batch's dtype).  Its kind is the network coupling's: chain_vjp_oracle hands every layer of that kind to the
    layer's own .vjp; nothing else reads the kind."""

    kind = "coupling_mlp"

    def __init__(self, W1, c1, W2, c2, deg=None, act="tanh", slope=0.0):
        H, D = np.shape(W1)
        self.args = (W1, c1, W2, c2, default_degrees(D, H) if deg is None else deg, act, slope)

    def forward(self, x):
        return forward(*self.args, x, np.asarray(x).dtype)

    def inverse(self, y):
        return inverse(*self.args, y, np.asarray(y).dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        x = np.asarray(x)
        return vjp(*self.args, x, ybar, ljbar, inverse, x.dtype)
