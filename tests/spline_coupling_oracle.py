"""Reference for the spline coupling layer, B2B_COUPLING_RQS: Coupling(x₂ -> RationalQuadraticSpline(…, B), mask)
(coupling.jl:206-228) whose knots come from the conditioner v = W·x₂ + c through the reference's normalising constructor
(rational_quadratic_spline.jl:109-123).  With n1 transformed rows and K bins, transformed row i takes

    raw widths v[i + n1·k] (k < K),  raw heights v[n1·K + i + n1·k] (k < K),  raw derivatives v[2·n1·K + i + n1·k] (k < K−1)

(0-based), i.e. reshape(v[1:n1K], n1, K) etc. in Julia's column-major order.

The forward and inverse are the generic oracle_np.coupling_forward / coupling_inverse, column by column, with a law object
over oracle_np.rqs_params / rqs_forward / rqs_inverse; ``dtype`` float32 evaluates the same formulas in float32, which
gives the reference's own float32 error for the parity gates.  ``vjp`` is the float64 reverse mode w.r.t. x, W and c:
the element cotangents of oracle_np.rqs_vjp pulled back through the normaliser (reverse cumsum, softmax pullback
ā = s ⊙ (s̄ − ⟨s̄, s⟩), r̄ = d̄·σ(r)), then x̄₂ = ȳ₂ + Wᵀr̄, W̄ = Σ r̄ x₂ᵀ, c̄ = Σ r̄."""
import numpy as np

from oracle import oracle_np as O


def raw_params(Wm, c, x2, K, dtype=np.float64):
    """(raw widths (n1, K), raw heights (n1, K), raw derivatives (n1, K−1)) of one column x₂ (n2,) or of a batch (n2, N),
    then with a trailing column axis."""
    dt = np.dtype(dtype)
    Wm = np.asarray(Wm, dt)
    J = 3 * K - 1
    n1 = Wm.shape[0] // J
    v = Wm @ np.asarray(x2, dt)
    if c is not None:
        v = v + (np.asarray(c, dt) if v.ndim == 1 else np.asarray(c, dt)[:, None])
    v = v.astype(dt)
    tail = v.shape[1:]
    rw = np.moveaxis(v[: n1 * K].reshape((K, n1) + tail), 0, 1)
    rh = np.moveaxis(v[n1 * K: 2 * n1 * K].reshape((K, n1) + tail), 0, 1)
    rd = np.moveaxis(v[2 * n1 * K:].reshape((K - 1, n1) + tail), 0, 1)
    return rw, rh, rd


class SplineLaw:
    """RationalQuadraticSpline with processed knots (n1 × K+1), as a coupling law (wladj / inv_wladj)."""

    def __init__(self, widths, heights, derivs):
        self.widths, self.heights, self.derivs = widths, heights, derivs

    def wladj(self, x1):
        return O.rqs_forward(self.widths, self.heights, self.derivs, np.asarray(x1))

    def inv_wladj(self, y1):
        return O.rqs_inverse(self.widths, self.heights, self.derivs, np.asarray(y1))


def spline_theta(Wm, c, K, B, dtype=np.float64):
    """θ(x₂) = RationalQuadraticSpline(reshape(W·x₂ + c …)..., B) with the reference's constructor."""

    def theta(x2):
        rw, rh, rd = raw_params(Wm, c, x2, K, dtype)
        return SplineLaw(*O.rqs_params(rw, rh, rd, B))

    return theta


def _mask(D, idx1, idx2):
    return O.PartitionMask.make(D, [int(i) for i in idx1], [int(i) for i in idx2])


def _run(step, idx1, idx2, Wm, c, K, B, x, dtype, cols):
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    D, N = x.shape
    cols = range(N) if cols is None else cols
    theta, mask = spline_theta(Wm, c, K, B, dt), _mask(D, idx1, idx2)
    ys, ljs = [], []
    for n in cols:
        y, lj = step(theta, mask, x[:, n])
        ys.append(y)
        ljs.append(np.asarray(lj).reshape(-1)[0])  # rqs_inverse returns a 1-vector for a vector input
    return np.stack(ys, axis=1).astype(dt), np.asarray(ljs, dt)


def forward(idx1, idx2, Wm, c, K, B, x, dtype=np.float64, cols=None):
    """with_logabsdet_jacobian(Coupling, x) for x (D, N) (or the columns ``cols``); idx1 / idx2 are 1-based row lists."""
    return _run(O.coupling_forward, idx1, idx2, Wm, c, K, B, x, dtype, cols)


def inverse(idx1, idx2, Wm, c, K, B, y, dtype=np.float64, cols=None):
    """with_logabsdet_jacobian(Inverse(Coupling), y)."""
    return _run(O.coupling_inverse, idx1, idx2, Wm, c, K, B, y, dtype, cols)


def vjp(idx1, idx2, Wm, c, K, B, x, ybar, ljbar, inverse=False, dtype=np.float64):
    """Reverse mode of forward (inverse=False) or inverse (inverse=True) at x (D, N; the observed y for the inverse):
    returns (x̄ (D, N), W̄ ((3K−1)n1, n2), c̄ ((3K−1)n1,)).  ybar (D, N) / ljbar (N,) may be None (zeros).  Float64 by
    default; float32 restates the same reverse sweep in float32 (the parity gates' own-error term)."""
    dt = np.dtype(dtype)
    x = np.asarray(x, dt)
    D, N = x.shape
    i1, i2 = np.asarray(idx1, int) - 1, np.asarray(idx2, int) - 1
    n1, n2 = len(i1), len(i2)
    Wm = np.asarray(Wm, dt)
    yb = np.zeros((D, N), dt) if ybar is None else np.asarray(ybar, dt)
    lb = np.zeros(N, dt) if ljbar is None else np.asarray(ljbar, dt)
    x1, x2 = x[i1], x[i2]
    rw, rh, rd = raw_params(Wm, c, x2, K, dt)  # (n1, K, N) ...
    # one "row" per (i, n): the element VJP of oracle_np.rqs_vjp with per-row knots, linear in (ȳ, l̄)
    flat = lambda a: np.moveaxis(a, 2, 1).reshape(n1 * N, a.shape[1])  # noqa: E731  (n1, k, N) -> (n1·N, k), row i·N + n
    fw, fh, fd = flat(rw), flat(rh), flat(rd)
    Wk, Hk, Dk = O.rqs_params(fw, fh, fd, B)
    xv = x1.reshape(n1 * N, 1)
    r1 = O.rqs_vjp(Wk, Hk, Dk, xv, yb[i1].reshape(n1 * N, 1), np.zeros(1, dt), inverse=inverse)
    r2 = O.rqs_vjp(Wk, Hk, Dk, xv, np.zeros((n1 * N, 1), dt), np.ones(1, dt), inverse=inverse)
    l_rows = np.repeat(lb[None, :], n1, axis=0).reshape(n1 * N, 1)
    x1b = r1[0] + l_rows * r2[0]
    Wb, Hb, Db = (a + l_rows * b for a, b in zip(r1[1:], r2[1:]))
    # pull back through the normaliser: knots = 2B·cumsum([0; softmax(a)]) − B, derivatives = [1; log1pexp(r); 1]
    def softmax_vjp(a, g):
        s = O.softmax_rows(a)
        sb = 2 * B * np.cumsum(g[:, :0:-1], axis=1)[:, ::-1]  # s̄_j = 2B Σ_{k > j} ḡ_k
        return s * (sb - np.sum(sb * s, axis=1, keepdims=True))
    aw, ah = softmax_vjp(fw, Wb), softmax_vjp(fh, Hb)
    ad = Db[:, 1:K] / (1 + np.exp(-fd))
    unflat = lambda a: np.moveaxis(a.reshape(n1, N, a.shape[1]), 1, 2)  # noqa: E731  -> (n1, k, N)
    rbar = np.concatenate([np.moveaxis(unflat(a), 1, 0).reshape(-1, N) for a in (aw, ah, ad)], axis=0)  # (J·n1, N)
    xbar = yb.copy()
    xbar[i1] = x1b.reshape(n1, N)
    xbar[i2] = yb[i2] + Wm.T @ rbar
    return xbar, (rbar @ x2.T).astype(dt), rbar.sum(axis=1, dtype=dt)


class SplineLayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse (evaluated in the batch's dtype)."""

    kind = "coupling_rqs"

    def __init__(self, idx1, idx2, Wm, c, K, B):
        self.idx1, self.idx2, self.Wm, self.c, self.K, self.B = idx1, idx2, Wm, c, K, B

    def forward(self, x):
        return forward(self.idx1, self.idx2, self.Wm, self.c, self.K, self.B, x, x.dtype)

    def inverse(self, y):
        return inverse(self.idx1, self.idx2, self.Wm, self.c, self.K, self.B, y, y.dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        x = np.asarray(x)
        xb, Wb, cb = vjp(self.idx1, self.idx2, self.Wm, self.c, self.K, self.B, x, ybar, ljbar, inverse, x.dtype)
        return xb, dict(W=Wb, c=cb)
