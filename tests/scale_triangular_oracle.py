"""Float64 restatement of the triangular Scale layer, B2B_SCALE_TRIANGULAR: Scale(T) with T one of LinearAlgebra's
LowerTriangular, UpperTriangular, UnitLowerTriangular or UnitUpperTriangular views of a D x D matrix (scale.jl:14,17,35-36:
`b.a * x`, `b.a \\ y`, `logabsdet(b.a)`, whose triangular arithmetic is LinearAlgebra's).

  M         the matrix the view stands for: the triangle of the stored T, the rest 0, a unit diagonal taken as 1
  forward   y = M x,      logjac = Σᵢ log|Tᵢᵢ|   (0 for the unit forms)
  inverse   y = M⁻¹ x     (a triangular solve), logjac = −Σᵢ log|Tᵢᵢ|
  reverse   u the layer's input, G = Σₙ ȳₙ uₙᵀ, s = Σₙ l̄ₙ, 𝒫 the entries of T the view reads (the triangle, strict for the
            unit forms); the dense layer's Ā projected on 𝒫:
            forward layer  x̄ = Mᵀ ȳ,     T̄ = 𝒫(G) + s·diag(1/Tᵢᵢ)
            inverse layer  x̄ = M⁻ᵀ ȳ,    T̄ = −𝒫(M⁻ᵀ G M⁻ᵀ) − s·diag(1/Tᵢᵢ)
            (no s term for the unit forms; T̄ is 0 outside 𝒫)
"""
import numpy as np
from scipy.linalg import solve_triangular

FORMS = [(False, False), (True, False), (False, True), (True, True)]  # (upper, unit)


def form_name(upper, unit):
    return ("Unit" if unit else "") + ("Upper" if upper else "Lower") + "Triangular"


def mask(D, upper, unit):
    """𝒫 as a boolean D x D matrix."""
    return np.triu(np.ones((D, D), bool), 1 if unit else 0) if upper else np.tril(np.ones((D, D), bool), -1 if unit else 0)


def view(T, upper, unit, dtype=np.float64):
    """The matrix M the triangular view of T stands for."""
    T = np.asarray(T, dtype)
    M = np.where(mask(T.shape[0], upper, unit), T, 0).astype(dtype)
    if unit:
        np.fill_diagonal(M, 1)
    return M


def logabsdet(T, upper, unit):
    return 0.0 if unit else float(np.sum(np.log(np.abs(np.diag(np.asarray(T, np.float64))))))


def forward(T, upper, unit, x, dtype=np.float64):
    x = np.asarray(x, dtype)
    return view(T, upper, unit, dtype) @ x, np.full(x.shape[1], logabsdet(T, upper, unit), dtype)


def inverse(T, upper, unit, y, dtype=np.float64):
    y = np.asarray(y, dtype)
    M = view(T, upper, unit, dtype)
    return solve_triangular(M, y, lower=not upper, unit_diagonal=unit), np.full(y.shape[1], -logabsdet(T, upper, unit), dtype)


def vjp(T, upper, unit, x, ybar, ljbar, inverse=False):
    """(x̄, T̄) of with_logabsdet_jacobian(Scale(view(T)), x) (inverse=False) or of its Inverse at x (D, N); ybar (D, N) /
    ljbar (N,) may be None (zeros)."""
    x = np.asarray(x, np.float64)
    D, N = x.shape
    M = view(T, upper, unit)
    yb = np.zeros((D, N)) if ybar is None else np.asarray(ybar, np.float64)
    s = 0.0 if ljbar is None else float(np.sum(np.asarray(ljbar, np.float64)))
    P = mask(D, upper, unit)
    dterm = np.zeros((D, D)) if unit else np.diag(1.0 / np.diag(np.asarray(T, np.float64)))
    G = yb @ x.T
    if not inverse:
        return M.T @ yb, np.where(P, G, 0) + s * dterm
    Bm = np.linalg.inv(M).T
    return Bm @ yb, np.where(P, -Bm @ G @ Bm, 0) - s * dterm


def random_tri(rng, D, upper, unit, dtype=np.float32):
    """T with diagonal ±U(0.5, 2) (about a quarter negative) and off-diagonal entries 0.3·N(0, 1)/√D: the views of it have
    a condition number of order 1 at every D (a unit triangle with N(0, 1) entries does not: it grows exponentially with D).
    The entries outside the view are N(0, 1), which the layer must never read."""
    T = rng.standard_normal((D, D))
    P = mask(D, upper, False)
    T = np.where(P, 0.3 * T / np.sqrt(D), T)
    d = rng.uniform(0.5, 2.0, D) * np.where(rng.uniform(size=D) < 0.25, -1.0, 1.0)
    np.fill_diagonal(T, d)
    return T.astype(dtype)


class TriLayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse and of chain_vjp_oracle.chain_vjp."""

    kind = "scale_matrix"  # chain_vjp_oracle differentiates layers of this kind by their own .vjp

    def __init__(self, T, upper, unit):
        self.T, self.upper, self.unit = np.asarray(T), upper, unit

    def forward(self, x):
        return forward(self.T, self.upper, self.unit, x, x.dtype)

    def inverse(self, y):
        return inverse(self.T, self.upper, self.unit, y, y.dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        xb, Tb = vjp(self.T, self.upper, self.unit, x, ybar, ljbar, inverse)
        return xb, dict(a=Tb)
