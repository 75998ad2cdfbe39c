"""Float64 restatement of the LU linear layer, B2B_SCALE_LU: LULinear(F, p), the map of
Permute(p) ∘ Scale(UnitLowerTriangular(F)) ∘ Scale(UpperTriangular(F)) as one layer.

  F         both factors packed as lu(A).factors: L = I + strict lower triangle of F, U = upper triangle with the diagonal
  P         (P v)[dst[r]] = v[r], dst = p − 1 (0-based; None: the identity)
  forward   y = P L U x,          logjac = Σᵢ log|Uᵢᵢ|
  inverse   y = U⁻¹ L⁻¹ Pᵀ x,     logjac = −Σᵢ log|Uᵢᵢ|
  reverse   u the layer's input, G = Σₙ ȳₙ uₙᵀ, s = Σₙ l̄ₙ, A = P L U;
            M̄ = G (forward layer) or −A⁻ᵀ G A⁻ᵀ (inverse layer), then through A = P L U:
            L̄ = 𝒮(Pᵀ M̄ Uᵀ),   Ū = 𝒰(Lᵀ Pᵀ M̄) ± s·diag(1/Uᵢᵢ)      (+ forward, − inverse; 𝒮 strict lower, 𝒰 upper)
            F̄ = L̄ + Ū, and x̄ = Aᵀ ȳ or A⁻ᵀ ȳ.
"""
import numpy as np
from scipy.linalg import solve_triangular


def factors(F):
    F = np.asarray(F, np.float64)
    return np.tril(F, -1) + np.eye(F.shape[0]), np.triu(F)


def perm_matrix(dst, D):
    """P with (P v)[dst[r]] = v[r]."""
    P = np.zeros((D, D))
    P[np.arange(D) if dst is None else np.asarray(dst), np.arange(D)] = 1.0
    return P


def matrix(F, dst):
    """A = P L U."""
    L, U = factors(F)
    return perm_matrix(dst, L.shape[0]) @ L @ U


def logabsdet(F):
    return float(np.sum(np.log(np.abs(np.diag(np.asarray(F, np.float64))))))


def forward(F, dst, x, dtype=np.float64):
    x = np.asarray(x, np.float64)
    y = matrix(F, dst) @ x
    return y.astype(dtype), np.full(x.shape[1], logabsdet(F), dtype)


def inverse(F, dst, y, dtype=np.float64):
    y = np.asarray(y, np.float64)
    L, U = factors(F)
    w = perm_matrix(dst, L.shape[0]).T @ y
    x = solve_triangular(U, solve_triangular(L, w, lower=True, unit_diagonal=True), lower=False)
    return x.astype(dtype), np.full(y.shape[1], -logabsdet(F), dtype)


def vjp(F, dst, x, ybar, ljbar, inverse=False):
    """(x̄, F̄) of with_logabsdet_jacobian(LULinear(F, dst + 1), x) (inverse=False) or of its Inverse at x (D, N); ybar (D, N)
    / ljbar (N,) may be None (zeros)."""
    x = np.asarray(x, np.float64)
    D, N = x.shape
    L, U = factors(F)
    P = perm_matrix(dst, D)
    A = P @ L @ U
    yb = np.zeros((D, N)) if ybar is None else np.asarray(ybar, np.float64)
    s = 0.0 if ljbar is None else float(np.sum(np.asarray(ljbar, np.float64)))
    G = yb @ x.T
    if not inverse:
        xb, Mb, sg = A.T @ yb, G, 1.0
    else:
        B = np.linalg.inv(A).T
        xb, Mb, sg = B @ yb, -B @ G @ B, -1.0
    Fb = np.tril(P.T @ Mb @ U.T, -1) + np.triu(L.T @ P.T @ Mb) + sg * s * np.diag(1.0 / np.diag(U))
    return xb, Fb


def random_lu(rng, D, dtype=np.float32):
    """F whose factors are well conditioned at every D: Uᵢᵢ = ±U(0.5, 2) (about a quarter negative), off-diagonal
    entries 0.3·N(0, 1)/√D in both triangles."""
    F = 0.3 * rng.standard_normal((D, D)) / np.sqrt(D)
    d = rng.uniform(0.5, 2.0, D) * np.where(rng.uniform(size=D) < 0.25, -1.0, 1.0)
    np.fill_diagonal(F, d)
    return F.astype(dtype)


class LULayer:
    """The layer as an element of oracle_np.chain_forward / chain_inverse and of chain_vjp_oracle.chain_vjp."""

    kind = "scale_matrix"  # chain_vjp_oracle differentiates layers of this kind by their own .vjp

    def __init__(self, F, dst):
        self.F, self.dst = np.asarray(F), dst

    def forward(self, x):
        return forward(self.F, self.dst, x, x.dtype)

    def inverse(self, y):
        return inverse(self.F, self.dst, y, y.dtype)

    def vjp(self, x, ybar, ljbar, inverse=False):
        xb, Fb = vjp(self.F, self.dst, x, ybar, ljbar, inverse)
        return xb, dict(factors=Fb)
