"""Float64 restatement of the dense Scale layer, B2B_SCALE_MATRIX: Scale(A) with a D x D matrix (scale.jl:14,17,35-36).

  forward   y = A x,       logjac = log|det A|   (logabsdet(A)[1], the same for every column)
  inverse   y = A⁻¹ y,     logjac = −log|det A|
  reverse   u the layer's input, G = Σₙ ȳₙ uₙᵀ, s = Σₙ l̄ₙ, B = A⁻ᵀ (d log|det A| / dA = A⁻ᵀ):
            forward layer  x̄ = Aᵀ ȳ,    Ā = G + s·B
            inverse layer  x̄ = A⁻ᵀ ȳ,   Ā = −B G B − s·B   (d(A⁻¹u) = −A⁻¹ dA A⁻¹ u)
"""
import numpy as np


def logabsdet(A):
    return float(np.linalg.slogdet(np.asarray(A, np.float64))[1])


def forward(A, x, dtype=np.float64):
    A, x = np.asarray(A, dtype), np.asarray(x, dtype)
    N = x.shape[1]
    return A @ x, np.full(N, logabsdet(A), dtype)


def inverse(A, y, dtype=np.float64):
    A, y = np.asarray(A, dtype), np.asarray(y, dtype)
    N = y.shape[1]
    return np.linalg.solve(A, y), np.full(N, -logabsdet(A), dtype)


def vjp(A, x, ybar, ljbar, inverse=False, dtype=np.float64):
    """(x̄, Ā) of with_logabsdet_jacobian(Scale(A), x) (inverse=False) or of Inverse(Scale(A)) (inverse=True) at x (D, N);
    ybar (D, N) / ljbar (N,) may be None (zeros).  Float64 by default; float32 restates the same formulas in float32 (the
    parity gates' own-error term)."""
    dt = np.dtype(dtype)
    A = np.asarray(A, dt)
    x = np.asarray(x, dt)
    D, N = x.shape
    yb = np.zeros((D, N), dt) if ybar is None else np.asarray(ybar, dt)
    s = dt.type(0) if ljbar is None else np.sum(np.asarray(ljbar, dt), dtype=dt)
    Bm = np.linalg.inv(A).T
    G = yb @ x.T
    if not inverse:
        return A.T @ yb, (G + s * Bm).astype(dt)
    return (Bm @ yb).astype(dt), (-Bm @ G @ Bm - s * Bm).astype(dt)


class ScaleLayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse (evaluated in the batch's dtype)."""

    kind = "scale_matrix"

    def __init__(self, A):
        self.A = np.asarray(A)

    def forward(self, x):
        return forward(self.A, x, x.dtype)

    def inverse(self, y):
        return inverse(self.A, y, y.dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        x = np.asarray(x)
        xb, Ab = vjp(self.A, x, ybar, ljbar, inverse, x.dtype)
        return xb, dict(a=Ab)


def well_conditioned(rng, D, scale=0.3):
    """A = I + scale·G/√D, G standard normal: condition number O(1) for every D."""
    return np.eye(D) + scale * rng.standard_normal((D, D)) / np.sqrt(D)
