"""The fused planar chain kernel at D = 128 (one thread per column, 32-column tiles, 8 warps per CTA): batches at and
around the tile width and the 256-column CTA round, batches that leave most warps of the grid without a tile (with the
columns behind the batch left untouched), and an inverse chain in which a single column takes the safeguarded find_alpha
fallback."""
import numpy as np
import pytest

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

D, RTOL = 128, 1e-5
f32 = np.float32


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(o32, o64, k=2.0):
    """1e-5 relative, or k times the float32 restatement's own error where that is larger (ill-conditioned inputs)."""
    return max(RTOL, k * rel(o32, o64))


def planar_layers(rng, L):
    out = []
    for _ in range(L):
        w, u = (rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32)
        b = rng.standard_normal(1).astype(f32)
        out.append((w, u, b))
    return out


def run_into_padded(B, flow, x, N):
    """run_chain into the first N columns of (D, N + 16) / (N + 16) buffers filled with a sentinel: the columns behind
    the batch must stay untouched."""
    import torch

    ybig = B.colmajor_empty(D, N + 16)
    ybig.fill_(7.0)
    ljbig = torch.full((N + 16,), 7.0, device="cuda")
    B.run_chain(flow, x, y=ybig[:, :N], logjac=ljbig[:N])
    assert bool((ybig[:, N:] == 7.0).all()) and bool((ljbig[N:] == 7.0).all())
    return B.to_numpy(ybig[:, :N]), B.to_numpy(ljbig[:N])


@pytest.mark.parametrize("N", [1, 15, 16, 17, 31, 32, 33, 255, 256, 257, 5000, 40000])
def test_planar_chain_batches_around_the_tile(B, N):
    """8 layers forward / inverse / logpdf with device- and host-resident parameters; N from one column (one tile, 7 of
    the 8 warps idle) over the 32-column tile and the 256-column CTA round to many CTAs with uneven tile counts."""
    rng = np.random.default_rng(N)
    params = planar_layers(rng, 8)
    olayers = [O.Layer("planar", dict(w=w, u=u, b=b)) for (w, u, b) in params]
    flow = B.Composed(*[B.PlanarLayer(w, u, b) for (w, u, b) in params])
    host_flow = B.Composed(*[B.PlanarLayer(w, u, b).to("cpu") for (w, u, b) in params])
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)

    y, lj = run_into_padded(B, flow, xd, N)
    assert B.lib().b2b_last_launch_count() == 1
    yo, ljo = O.chain_forward(olayers, x.astype(np.float64))
    assert rel(y, yo) <= RTOL and rel(lj, ljo) <= RTOL, (rel(y, yo), rel(lj, ljo))
    lib = B.lib()
    try:  # the layer interpreter, an independent program over the same descriptors
        assert lib.b2b_set_kernel_variant(2) == 0
        yi, lji = run_into_padded(B, flow, xd, N)
    finally:
        lib.b2b_set_kernel_variant(0)
    assert rel(y, yi) <= 5e-6 and rel(lj, lji) <= 5e-6
    yh, ljh = run_into_padded(B, host_flow, xd, N)
    assert rel(y, yh) <= 2e-6 and rel(lj, ljh) <= 2e-6

    yd = B.from_numpy(y)
    inv = B.inverse(flow)
    xi, ljinv = run_into_padded(B, inv, yd, N)
    xo, ljio = O.chain_inverse(olayers, y.astype(np.float64))
    xo32, ljio32 = O.chain_inverse(olayers, y)
    assert rel(xi, xo) <= gate(xo32, xo) and rel(ljinv, ljio) <= gate(ljio32, ljio)
    xh, ljih = run_into_padded(B, B.inverse(host_flow), yd, N)
    assert rel(xi, xh) <= 5e-6 and rel(ljinv, ljih) <= 5e-6

    td = B.transformed(B.MvNormal(D), flow)
    total, lp = B.logpdf_sum(td, yd)
    lpo = O.mvnormal_diag_logpdf(None, None, xo) + ljio  # logpdf(td, y) = logpdf(base, x) + logabsdetjac(inverse, y)
    assert rel(B.to_numpy(lp), lpo) <= RTOL
    assert abs(float(total) - float(lpo.sum())) <= 1e-5 * max(abs(float(lpo.sum())), 1.0)


@pytest.mark.parametrize("col", [0, 5, 31, 32 + 9])
def test_planar_inverse_fallback_in_one_column(B, col):
    """The last forward layer has wᵀû = -0.999, where the root G_c(s) of u + c·tanh u = s has a slope of 1000 at s = 0:
    the tabulated root is not trusted there and the whole warp takes the safeguarded iteration.  Every column of the
    batch but `col` gets s in [2, 4]; column `col` gets s = 0.01, so ONE column of one warp forces the fallback, and
    every row of that column must be updated with the same tanh."""
    rng = np.random.default_rng(40 + col)
    N = 64
    params = planar_layers(rng, 3)
    w, _, b = params[-1]
    c = -0.999
    wu = np.log(np.expm1(c + 1.0))  # wᵀu whose wᵀû = softplus(wᵀu) − 1 = c (planar_layer.jl:65-70)
    w64 = w.astype(np.float64)
    u = rng.standard_normal(D)
    u = (u - w64 * (w64 @ u) / (w64 @ w64) + w64 * wu / (w64 @ w64)).astype(f32)
    params[-1] = (w, u, b)
    olayers = [O.Layer("planar", dict(w=w_, u=u_, b=b_)) for (w_, u_, b_) in params]
    flow = B.Composed(*[B.PlanarLayer(w_, u_, b_) for (w_, u_, b_) in params])
    host_flow = B.Composed(*[B.PlanarLayer(w_, u_, b_).to("cpu") for (w_, u_, b_) in params])

    s = rng.uniform(2.0, 4.0, N)
    s[col] = 0.01
    z = rng.standard_normal((D, N))
    z = z - np.outer(w64, w64 @ z) / (w64 @ w64) + np.outer(w64, s - float(b[0])) / (w64 @ w64)
    y = z.astype(f32)
    yd = B.from_numpy(y)

    # the layer alone: inverse(y) = y − û·tanh(α+b) (planar_layer.jl:124); the tanh recovered from each half
    x1 = B.to_numpy(B.inverse(B.PlanarLayer(w, u, b))(yd)).astype(np.float64)
    wu32 = float(w64 @ u.astype(np.float64))
    uhat = u + (np.log1p(np.exp(-wu32)) - 1.0) * w64 / (w64 @ w64)  # get_u_hat, planar_layer.jl:65-70
    d = y[:, col].astype(np.float64) - x1[:, col]
    t_lo, t_hi = (uhat[h] @ d[h] / (uhat[h] @ uhat[h]) for h in (slice(0, 64), slice(64, 128)))
    assert t_lo > 0.05 and abs(t_lo - t_hi) <= 1e-4 * abs(t_lo), (t_lo, t_hi)

    xi, lji = B.with_logabsdet_jacobian(B.inverse(flow), yd)
    xi, lji = B.to_numpy(xi), B.to_numpy(lji)
    xo, ljio = O.chain_inverse(olayers, y.astype(np.float64))
    xo32, ljio32 = O.chain_inverse(olayers, y)
    assert rel(xi, xo) <= gate(xo32, xo) and rel(lji, ljio) <= gate(ljio32, ljio), (rel(xi, xo), rel(lji, ljio))
    # host-resident parameters take the safeguarded iteration for every column (no root table)
    xh, ljh = B.with_logabsdet_jacobian(B.inverse(host_flow), yd)
    assert rel(xi, B.to_numpy(xh)) <= 5e-6 and rel(lji, B.to_numpy(ljh)) <= 5e-6
