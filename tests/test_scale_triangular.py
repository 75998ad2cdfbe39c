"""GPU tests of the triangular Scale layer, B2B_SCALE_TRIANGULAR: Scale(T) with T a LowerTriangular, UpperTriangular,
UnitLowerTriangular or UnitUpperTriangular view, against the float64 restatement of tests/scale_triangular_oracle.py.  y is
held to the dense layer's componentwise bound, (4·D + 2)·eps32·(|M||x|) with M the view (forward) or its inverse (times
the asserted condition number), and the log-Jacobian to about 1e-6·D."""
import numpy as np
import pytest

import chain_vjp_oracle as V
import elementwise_vec_oracle as E
import rsample_oracle as R
import scale_triangular_oracle as S
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
EPS = float(np.finfo(f32).eps)
COND_MAX = 20.0
FORM_IDS = [S.form_name(u, n) for u, n in S.FORMS]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def tri(rng, D, upper, unit):
    T = S.random_tri(rng, D, upper, unit)
    if D >= 2:
        assert np.linalg.cond(S.view(T, upper, unit)) < COND_MAX
    return T


def layer(B, T, upper, unit, **kw):
    return B.Scale(getattr(B, S.form_name(upper, unit))(T), **kw)


def check_y(y, M, x, inv):
    M64, x64 = M.astype(np.float64), x.astype(np.float64)
    Mi = np.linalg.inv(M64) if inv else M64
    bound = (4 * M.shape[0] + 2) * EPS * (np.abs(Mi) @ np.abs(x64)) * (COND_MAX if inv else 1.0) + 1e-30
    err = np.abs(np.asarray(y, np.float64) - Mi @ x64)
    assert (err <= bound).all(), float((err / bound).max())


def check_lj(lj, T, upper, unit, inv):
    want = S.logabsdet(T, upper, unit) * (-1 if inv else 1)
    assert np.abs(np.asarray(lj, np.float64) - want).max() <= 1e-6 * T.shape[0] + 2e-7 * abs(want) + 1e-6


SHAPES = [(1, 1), (2, 0), (3, 1001), (17, 129), (32, 1000), (64, (1 << 19) + 3), (100, 333), (128, 4099), (255, 257),
          (256, 1000)]


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("upper,unit", S.FORMS, ids=FORM_IDS)
@pytest.mark.parametrize("D,N", SHAPES)
def test_parity(B, D, N, upper, unit, inv):
    rng = np.random.default_rng(D * 13 + N % 1000 + 7 * inv + 3 * upper + 5 * unit)
    T = tri(rng, D, upper, unit)
    x = rng.standard_normal((D, N)).astype(f32)
    lay = layer(B, T, upper, unit)
    xd = B.from_numpy(x) if N else B.colmajor_empty(D, 0, "cuda")
    y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, xd)
    assert tuple(y.shape) == (D, N) and tuple(lj.shape) == (N,)
    if N == 0:
        return
    check_y(B.to_numpy(y), S.view(T, upper, unit), x, inv)
    check_lj(B.to_numpy(lj), T, upper, unit, inv)


def _raw(B, lay, inv, D, N, x, ldx, xoff, y, ldy, yoff, lj, acc):
    import torch

    from bijectors_jl_b200.interface import _desc_array, _stream

    arr = _desc_array(lay._descs(inv, D))
    L = B.lib()
    wsb = L.b2b_chain_workspace_bytes(arr, 1, D, N, 1 if y is not None else 0, 0)
    assert wsb > 0
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    p = lambda t, off: None if t is None else t.data_ptr() + 4 * off  # noqa: E731
    rc = L.b2b_chain_run_f32(arr, 1, p(x, xoff), p(y, yoff), p(lj, 0), None, D, N, ldx, ldy, acc, ws.data_ptr(), wsb,
                             _stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("upper,unit", S.FORMS, ids=FORM_IDS)
@pytest.mark.parametrize("D", [5, 130])
def test_unread_entries_and_call_modes(B, D, upper, unit, inv):
    """NaN in every entry the view does not read gives the bits of zeros there; padded ld and offset bases, accumulate,
    y == NULL, in place, repeats and a shorter batch give the bits of the plain call."""
    import torch

    rng = np.random.default_rng(11 + inv + D + 2 * upper + 4 * unit)
    N = 333
    T = tri(rng, D, upper, unit)
    read = S.mask(D, upper, unit) | (np.eye(D, dtype=bool) & (not unit))
    Tz, Tn = np.where(read, T, 0).astype(f32), np.where(read, T, np.nan).astype(f32)
    x = rng.standard_normal((D, N)).astype(f32)
    lay = layer(B, Tn, upper, unit)
    t = B.inverse(lay) if inv else lay
    lz = layer(B, Tz, upper, unit)
    y0, l0 = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(t, B.from_numpy(x)))
    yz, lz_ = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(B.inverse(lz) if inv else lz, B.from_numpy(x)))
    assert y0.tobytes() == yz.tobytes() and l0.tobytes() == lz_.tobytes() and np.isfinite(y0).all()
    y1, l1 = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(t, B.from_numpy(x)))
    assert y1.tobytes() == y0.tobytes() and l1.tobytes() == l0.tobytes()
    ys, _ = B.with_logabsdet_jacobian(t, B.from_numpy(x[:, :57].copy()))
    assert B.to_numpy(ys).tobytes() == y0[:, :57].copy().tobytes()  # a column does not depend on N
    ld, sentinel = D + 3, 7.25
    xb = torch.full((ld * N + 8,), sentinel, device="cuda")
    xv = xb[1:1 + ld * N].view(N, ld)
    xv[:, :D] = torch.from_numpy(x.T.copy()).cuda()
    yb = torch.full((ld * N + 8,), sentinel, device="cuda")
    lj = torch.empty(N, device="cuda")
    assert _raw(B, lay, inv, D, N, xb, ld, 1, yb, ld, 3, lj, 0) == 0
    yv = yb[3:3 + ld * N].view(N, ld)
    assert yv[:, :D].cpu().numpy().T.tobytes() == y0.tobytes()
    assert (yv[:, D:] == sentinel).all() and (yb[:3] == sentinel).all()
    assert lj.cpu().numpy().tobytes() == l0.tobytes()
    base = torch.randn(N, device="cuda")
    lj.copy_(base)
    assert _raw(B, lay, inv, D, N, xb, ld, 1, yb, ld, 3, lj, 1) == 0
    assert lj.cpu().numpy().tobytes() == (base.cpu().numpy() + l0).astype(f32).tobytes()
    lj.fill_(0)
    assert _raw(B, lay, inv, D, N, xb, ld, 1, None, D, 0, lj, 0) == 0
    assert lj.cpu().numpy().tobytes() == l0.tobytes()
    assert _raw(B, lay, inv, D, N, xb, ld, 1, xb, ld, 1, lj, 0) == 0  # in place
    assert xv[:, :D].cpu().numpy().T.tobytes() == y0.tobytes()
    assert (xv[:, D:] == sentinel).all() and lj.cpu().numpy().tobytes() == l0.tobytes()


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("upper,unit", S.FORMS, ids=FORM_IDS)
def test_agrees_with_the_dense_layer(B, upper, unit, inv):
    import torch

    rng = np.random.default_rng(23 + inv + 2 * upper + 4 * unit)
    D, N = 96, 3000
    T = tri(rng, D, upper, unit)
    M = S.view(T, upper, unit).astype(f32)
    x = rng.standard_normal((D, N)).astype(f32)
    yb = rng.standard_normal((D, N)).astype(f32)
    lb = torch.randn(N, device="cuda")
    lt, ld = layer(B, T, upper, unit), B.Scale(M)
    tt, td = (B.inverse(lt), B.inverse(ld)) if inv else (lt, ld)
    y_t, l_t = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(tt, B.from_numpy(x)))
    y_d, l_d = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(td, B.from_numpy(x)))
    check_y(y_t, M, x, inv)
    bound = 2 * (4 * D + 2) * EPS * (np.abs(np.linalg.inv(M.astype(np.float64)) if inv else np.abs(M)) @ np.abs(x)) * \
        (COND_MAX if inv else 1.0)
    assert (np.abs(y_t.astype(np.float64) - y_d) <= bound + 1e-30).all()
    assert np.abs(l_t.astype(np.float64) - l_d).max() <= 1e-6 * D
    _, g_t = B.chain_vjp(tt, B.from_numpy(x), B.from_numpy(yb), lb)
    _, g_d = B.chain_vjp(td, B.from_numpy(x), B.from_numpy(yb), lb)
    P = S.mask(D, upper, unit)
    Ab = np.where(P, g_d[0]["a"].cpu().numpy(), 0)
    assert rel(g_t[0]["a"].cpu().numpy(), Ab) < 2e-4


VJP_SHAPES = [(1, 50), (3, 1001), (64, 20000), (200, 3000), (256, 1500)]


@pytest.mark.parametrize("yb,ljb", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("upper,unit", S.FORMS, ids=FORM_IDS)
@pytest.mark.parametrize("D,N", VJP_SHAPES)
def test_vjp(B, D, N, upper, unit, inv, yb, ljb):
    import torch

    rng = np.random.default_rng(D + N + 2 * inv + 4 * yb + 8 * ljb + 16 * upper + 32 * unit)
    T = tri(rng, D, upper, unit)
    x = rng.standard_normal((D, N)).astype(f32)
    ybar = rng.standard_normal((D, N)).astype(f32) if yb else None
    lbar = rng.standard_normal(N).astype(f32) if ljb else None
    lay = layer(B, T, upper, unit)
    t = B.inverse(lay) if inv else lay
    xbar, grads = B.chain_vjp(t, B.from_numpy(x), None if ybar is None else B.from_numpy(ybar),
                              None if lbar is None else torch.from_numpy(lbar).cuda())
    xb64, Tb64 = S.vjp(T, upper, unit, x, ybar, lbar, inverse=inv)
    xb = B.to_numpy(xbar)
    if yb:
        check_y(xb, S.view(T, upper, unit).T.astype(f32), ybar, inv)
    else:
        assert not xb.any()
    Tb = grads[0]["a"].cpu().numpy()
    assert not Tb[~S.mask(D, upper, unit)].any()  # exactly 0 outside 𝒫
    if unit and not yb or D == 1 and unit:
        assert not Tb.any()
    else:
        assert rel(Tb, Tb64) < 2e-4, rel(Tb, Tb64)


def _flow(B, rng, D):
    """Permute ∘ Scale(UnitLowerTriangular) ∘ Scale(UpperTriangular) ∘ vector Shift ∘ vector Scale ∘ Coupling, device
    and oracle layers, inner-most first."""
    dev, ora = [], []
    n1 = D // 2
    cW = (rng.standard_normal((2 * n1, D - n1)) * 0.05).astype(f32)
    cc = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    i1, i2 = list(range(1, n1 + 1)), list(range(n1 + 1, D + 1))
    dev.append(B.Coupling(B.AffineConditioner(cW, cc), B.PartitionMask(D, i1, i2)))
    ora.append(O.Layer("coupling_affine", dict(idx1=np.asarray(i1), idx2=np.asarray(i2), W=cW, c=cc)))
    a = rng.uniform(0.7, 1.4, D).astype(f32)
    dev.append(B.Scale(a))
    ora.append(E.VecLayer(E.SCALE, a))
    b = (rng.standard_normal(D) * 0.2).astype(f32)
    dev.append(B.Shift(b))
    ora.append(E.VecLayer(E.SHIFT, b))
    U = tri(rng, D, True, False)
    dev.append(layer(B, U, True, False))
    ora.append(S.TriLayer(U, True, False))
    L = tri(rng, D, False, True)
    dev.append(layer(B, L, False, True))
    ora.append(S.TriLayer(L, False, True))
    perm = rng.permutation(D) + 1
    dev.append(B.Permute(perm))
    ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))))
    return B.Composed(*dev), ora


def test_chain_logpdf_and_vjp(B):
    import torch

    rng = np.random.default_rng(31)
    D, N = 32, 4000
    flow, ora = _flow(B, rng, D)
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.3, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu=mu, sigma=sigma), flow)
    y = (rng.standard_normal((D, N)) * 0.8).astype(f32)
    yd = B.from_numpy(y)
    lp = B.to_numpy(B.logpdf(td, yd))
    inv_layers, flags = ora[::-1], [True] * len(ora)
    _, lp64 = V.chain_logjac(inv_layers, flags, y.astype(np.float64), mu, sigma, terminal=True)
    assert rel(lp, lp64) < 1e-5
    lb = rng.standard_normal(N)
    ybar, fgrads, bgrads = B.logpdf_vjp(td, yd, torch.from_numpy(lb.astype(f32)).cuda())
    g, grads, base = E.chain_vjp(inv_layers, flags, y, None, lb, mu, sigma, terminal=True)
    assert rel(B.to_numpy(ybar), g) < 1e-4
    flow_grads = grads[::-1]
    for k in range(1, 5):
        assert rel(fgrads[k]["a"].cpu().numpy(), flow_grads[k]["a"]) < 1e-4, k
    for k in (3, 4):
        P = S.mask(D, *((True, False) if k == 3 else (False, True)))
        assert not fgrads[k]["a"].cpu().numpy()[~P].any()
    assert rel(bgrads["σ"].cpu().numpy(), base["σ"]) < 1e-4


def test_rand_vjp_through_the_layer(B):
    import torch

    rng = np.random.default_rng(41)
    D, N, SEED = 48, 6000, 1234
    T = tri(rng, D, False, False)
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.3, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu=mu, sigma=sigma), layer(B, T, False, False))
    ybar = torch.from_numpy(rng.standard_normal((D, N)).astype(f32)).cuda()
    qbar = torch.from_numpy(rng.standard_normal(N).astype(f32)).cuda()
    fg, bg = B.rand_vjp(td, N, B.from_numpy(ybar.cpu().numpy()), qbar, seed=SEED)
    z = O.philox_normals(SEED, 0, D, N)
    x = B.to_numpy(B.rand(td.dist, N, seed=SEED))
    g64, b64 = R.vjp([S.TriLayer(T, False, False)], [False], z, ybar.cpu().numpy(), qbar.cpu().numpy(), mu, sigma, x=x)
    assert rel(fg[0]["a"].cpu().numpy(), g64[0]["a"]) < 2e-4
    assert rel(bg["μ"].cpu().numpy(), b64["μ"]) < 2e-4 and rel(bg["σ"].cpu().numpy(), b64["σ"]) < 2e-4


def test_graph_replay_and_determinism(B):
    import torch

    rng = np.random.default_rng(61)
    D, N = 128, 20000
    flow, _ = _flow(B, rng, D)
    x = B.from_numpy((rng.standard_normal((D, N)) * 0.8).astype(f32))
    yb = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lb = torch.randn(N, device="cuda")
    r1 = B.with_logabsdet_jacobian(flow, x)
    a = B.chain_vjp(flow, x, yb, lb)
    b = B.chain_vjp(flow, x, yb, lb)
    assert torch.equal(a[0], b[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], b[1]) for k in p)
    out = {}
    g = B.GraphedCalls(lambda: out.__setitem__("r", (B.with_logabsdet_jacobian(B.inverse(flow), r1[0]),
                                                      B.chain_vjp(flow, x, yb, lb))))
    inv_eager = B.with_logabsdet_jacobian(B.inverse(flow), r1[0])
    (fi, cr) = out["r"]
    fi[0].fill_(float("nan"))
    cr[0].fill_(float("nan"))
    g()
    torch.cuda.synchronize()
    assert torch.equal(fi[0], inv_eager[0]) and torch.equal(fi[1], inv_eager[1])
    assert torch.equal(a[0], cr[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], cr[1]) for k in p)


def test_lu_pair_matches_the_dense_product(B):
    """Scale(UnitLowerTriangular(L)) ∘ Scale(UpperTriangular(U)) is Scale(L·U), both directions."""
    rng = np.random.default_rng(71)
    D, N = 256, 4000
    L, U = tri(rng, D, False, True), tri(rng, D, True, False)
    A = (S.view(L, False, True) @ S.view(U, True, False)).astype(f32)
    assert np.linalg.cond(A.astype(np.float64)) < COND_MAX * COND_MAX
    pair = B.Composed(layer(B, U, True, False), layer(B, L, False, True))
    x = rng.standard_normal((D, N)).astype(f32)
    for inv in (False, True):
        tp, td = (B.inverse(pair), B.inverse(B.Scale(A))) if inv else (pair, B.Scale(A))
        y_p, l_p = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(tp, B.from_numpy(x)))
        y_d, l_d = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(td, B.from_numpy(x)))
        want = np.linalg.solve(A.astype(np.float64), x) if inv else A.astype(np.float64) @ x
        assert rel(y_p, want) < 1e-5 and rel(y_d, want) < 1e-5
        assert np.abs(l_p.astype(np.float64) - l_d).max() <= 1e-5 * D


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("upper,unit", S.FORMS, ids=FORM_IDS)
@pytest.mark.parametrize("D,N", [(7, 300), (300, 200), (2048, 24)])
def test_float64(B, D, N, upper, unit, inv):
    import torch

    rng = np.random.default_rng(D + 2 * inv + 4 * upper + 8 * unit)
    T = S.random_tri(rng, D, upper, unit, np.float64)
    T[~(S.mask(D, upper, unit) | (np.eye(D, dtype=bool) & (not unit)))] = np.nan  # never read, the unit diagonal included
    x, ybar, lbar = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    lay = layer(B, T, upper, unit, dtype=torch.float64)
    t = B.inverse(lay) if inv else lay
    xd = B.from_numpy(x, dtype=np.float64)
    y, lj = B.with_logabsdet_jacobian(t, xd)
    y64, l64 = (S.inverse if inv else S.forward)(T, upper, unit, x)
    assert rel(B.to_numpy(y), y64) < 1e-12 and np.abs(B.to_numpy(lj) - l64).max() <= 1e-12 * max(1.0, abs(l64[0]))
    xbar, grads = B.chain_vjp(t, xd, B.from_numpy(ybar, dtype=np.float64), torch.from_numpy(lbar).cuda())
    xb64, Tb64 = S.vjp(T, upper, unit, x, ybar, lbar, inverse=inv)
    Tb = grads[0]["a"].cpu().numpy()
    assert rel(B.to_numpy(xbar), xb64) < 1e-12 and rel(Tb, Tb64) < 1e-12
    assert not Tb[~S.mask(D, upper, unit)].any()


def test_training_fits_the_covariance_and_keeps_the_unread_triangle(B):
    """Flow(Scale(LowerTriangular(L₀)), MvNormal(D)) fitted by Adam to Gaussian data: L Lᵀ reaches the sample covariance,
    and the parameter's upper-triangle entries keep their bits through every step (T̄ is exactly 0 there)."""
    import torch

    rng = np.random.default_rng(81)
    D, N = 6, 20000
    Lstar = np.tril(rng.standard_normal((D, D)) * 0.3) + np.diag(rng.uniform(0.6, 1.5, D))
    data = (Lstar @ rng.standard_normal((D, N))).astype(f32)
    C = np.cov(data.astype(np.float64), bias=True)
    L0 = np.eye(D, dtype=f32) + np.triu(np.full((D, D), 5.0, f32), 1)  # unread entries: any value
    sc = B.Scale(B.LowerTriangular(L0))
    flow = B.autograd.Flow(sc, B.MvNormal(D))
    (p,) = [q for q in flow.params if q.shape == (D, D)]
    upper0 = p.detach().t().triu(1).clone()
    y = B.from_numpy(data)
    opt = torch.optim.Adam(flow.parameters(), lr=3e-2)
    for _ in range(400):
        opt.zero_grad()
        flow.nll(y).backward()
        opt.step()
        assert torch.equal(p.detach().t().triu(1), upper0)
    Lf = np.tril(p.detach().t().cpu().numpy().astype(np.float64))
    assert rel(Lf @ Lf.T, C) < 0.05, rel(Lf @ Lf.T, C)
