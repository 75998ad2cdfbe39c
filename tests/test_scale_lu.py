"""GPU tests of the LU linear layer, B2B_SCALE_LU: LULinear(F, p) against the float64 restatement of
tests/scale_lu_oracle.py.  y is held to the dense layer's componentwise bound, (4·D + 2)·eps32·(|M||x|) with M = P·L·U
(forward) or its inverse (times the asserted condition number), and the log-Jacobian to about 1e-6·D."""
import numpy as np
import pytest

import coupling_mlp_rqs_oracle as C
import elementwise_vec_oracle as E
import rsample_oracle as R
import scale_lu_oracle as S
import scale_triangular_oracle as T
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
EPS = float(np.finfo(f32).eps)
COND_MAX = 20.0


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def lu_params(rng, D, perm):
    """(F, dst, p): F from S.random_lu, dst the 0-based destination rows (None for perm == "null"), p the 1-based
    indices LULinear takes (None, the identity or a random permutation)."""
    F = S.random_lu(rng, D)
    if D >= 2:
        assert np.linalg.cond(S.matrix(F, None)) < COND_MAX
    if perm == "null":
        return F, None, None
    dst = np.arange(D) if perm == "identity" else rng.permutation(D)
    return F, dst, dst + 1


def check_y(y, A, x, inv, cols=None):
    A64 = A.astype(np.float64)
    Mi = np.linalg.inv(A64) if inv else A64
    x64 = x.astype(np.float64) if cols is None else x[:, cols].astype(np.float64)
    y = np.asarray(y, np.float64) if cols is None else np.asarray(y, np.float64)[:, cols]
    bound = (4 * A.shape[0] + 2) * EPS * (np.abs(Mi) @ np.abs(x64)) * (COND_MAX if inv else 1.0) + 1e-30
    err = np.abs(y - Mi @ x64)
    assert (err <= bound).all(), float((err / bound).max())


def check_lj(lj, F, inv):
    want = S.logabsdet(F) * (-1 if inv else 1)
    assert np.abs(np.asarray(lj, np.float64) - want).max() <= 1e-6 * F.shape[0] + 2e-7 * abs(want) + 1e-6


PERMS = ["null", "identity", "random"]


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("perm", PERMS)
@pytest.mark.parametrize("N", [1, 1000, (1 << 20) + 13])
@pytest.mark.parametrize("D", [1, 2, 31, 32, 33, 64, 100, 128, 255, 256])
def test_parity(B, D, N, perm, inv):
    rng = np.random.default_rng(D * 13 + N % 1000 + 7 * inv + 3 * PERMS.index(perm))
    F, dst, p = lu_params(rng, D, perm)
    x = rng.standard_normal((D, N), dtype=f32)
    lay = B.LULinear(F, p)
    y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, B.from_numpy(x))
    assert tuple(y.shape) == (D, N) and tuple(lj.shape) == (N,)
    # at the large N the oracle checks 4096 spread columns and the ragged tail; the log-Jacobian is checked everywhere
    cols = None if N <= 1000 else np.unique(np.concatenate([np.linspace(0, N - 1, 4096).astype(np.int64),
                                                             np.arange(N - 13, N)]))
    check_y(B.to_numpy(y), S.matrix(F, dst), x, inv, cols)
    check_lj(B.to_numpy(lj), F, inv)


def test_launch_count(B):
    """One layer, either direction: the prep launch and the map."""
    rng = np.random.default_rng(3)
    D, N = 128, 5000
    F, _, p = lu_params(rng, D, "random")
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lay = B.LULinear(F, p)
    for t in (lay, B.inverse(lay)):
        B.with_logabsdet_jacobian(t, x)
        assert B.lib().b2b_last_launch_count() == 2


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
@pytest.mark.parametrize("D", [5, 130])
def test_call_modes(B, D, inv):
    """Padded ld and offset bases, accumulate, y == NULL, in place, repeats and a shorter batch give the bits of the plain
    call."""
    import torch

    rng = np.random.default_rng(11 + inv + D)
    N = 333
    F, _, p = lu_params(rng, D, "random")
    x = rng.standard_normal((D, N)).astype(f32)
    lay = B.LULinear(F, p)
    t = B.inverse(lay) if inv else lay
    y0, l0 = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(t, B.from_numpy(x)))
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


@pytest.mark.parametrize("D", [32, 96, 256])
def test_agrees_with_the_composition_and_the_dense_layer(B, D):
    """LULinear.from_matrix(A) against Permute(p) ∘ Scale(UnitLowerTriangular(F)) ∘ Scale(UpperTriangular(F)) and against
    Scale(A), both directions and reverse mode, each within the float32 gate of the float64 result."""
    import torch

    rng = np.random.default_rng(23 + D)
    N = 3000
    Q, _ = np.linalg.qr(rng.standard_normal((D, D)))
    A = (Q @ np.diag(rng.uniform(0.7, 1.4, D))).astype(f32)  # a random rotation, scaled
    lay = B.LULinear.from_matrix(A)
    F, p = lay.factors.cpu().numpy(), lay.p
    comp = B.Composed(B.Scale(B.UpperTriangular(F)), B.Scale(B.UnitLowerTriangular(F)), B.Permute(p))
    dense = B.Scale(A)
    A_lu = S.matrix(F, p - 1)
    assert rel(A_lu, A) < 1e-6
    x = rng.standard_normal((D, N)).astype(f32)
    yb = rng.standard_normal((D, N)).astype(f32)
    lb = torch.randn(N, device="cuda")
    for inv in (False, True):
        ts = [B.inverse(t) if inv else t for t in (lay, comp, dense)]
        outs = [[B.to_numpy(a) for a in B.with_logabsdet_jacobian(t, B.from_numpy(x))] for t in ts]
        for (y, lj), M in zip(outs, (A_lu, A_lu, A.astype(np.float64))):
            check_y(y, M, x, inv)
            check_lj(lj, F, inv)
        xb64, Fb64 = S.vjp(F, p - 1, x, yb, lb.cpu().numpy(), inverse=inv)
        xbar, g = B.chain_vjp(ts[0], B.from_numpy(x), B.from_numpy(yb), lb)
        assert rel(B.to_numpy(xbar), xb64) < 2e-5 and rel(g[0]["factors"].cpu().numpy(), Fb64) < 2e-4
        xc, gc = B.chain_vjp(ts[1], B.from_numpy(x), B.from_numpy(yb), lb)
        assert rel(B.to_numpy(xc), B.to_numpy(xbar)) < 4e-5
        # the composition's two triangular cotangents are the two halves of F̄
        U_c, L_c = (gc[0] if not inv else gc[2])["a"].cpu().numpy(), (gc[1])["a"].cpu().numpy()
        assert rel(np.tril(L_c, -1) + np.triu(U_c), g[0]["factors"].cpu().numpy()) < 4e-4


VJP_SHAPES = [(1, 50), (3, 1001), (64, 20000), (200, 3000), (256, 1500)]


@pytest.mark.parametrize("yb,ljb", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("perm", ["null", "random"])
@pytest.mark.parametrize("D,N", VJP_SHAPES)
def test_vjp(B, D, N, perm, inv, yb, ljb):
    import torch

    rng = np.random.default_rng(D + N + 2 * inv + 4 * yb + 8 * ljb + 16 * (perm == "random"))
    F, dst, p = lu_params(rng, D, perm)
    x = rng.standard_normal((D, N)).astype(f32)
    ybar = rng.standard_normal((D, N)).astype(f32) if yb else None
    lbar = rng.standard_normal(N).astype(f32) if ljb else None
    lay = B.LULinear(F, p)
    t = B.inverse(lay) if inv else lay
    xbar, grads = B.chain_vjp(t, B.from_numpy(x), None if ybar is None else B.from_numpy(ybar),
                              None if lbar is None else torch.from_numpy(lbar).cuda())
    xb64, Fb64 = S.vjp(F, dst, x, ybar, lbar, inverse=inv)
    xb = B.to_numpy(xbar)
    if yb:
        check_y(xb, S.matrix(F, dst).T.astype(f32), ybar, inv)
    else:
        assert not xb.any()
    assert rel(grads[0]["factors"].cpu().numpy(), Fb64) < 2e-4


def _spline_flow(B, rng, D):
    """Coupling(MLPSplineConditioner) ∘ LULinear ∘ Coupling(MLPSplineConditioner) ∘ LULinear, device and oracle layers,
    inner-most first."""
    dev, ora = [], []
    K, Bv, H = 5, 3.0, 16
    for k in range(2):
        F, dst, p = lu_params(rng, D, "random")
        dev.append(B.LULinear(F, p))
        ora.append(S.LULayer(F, dst))
        rows = rng.permutation(D) + 1
        n1 = D // 2
        idx1, idx2 = [int(i) for i in rows[:n1]], [int(i) for i in rows[n1:]]
        J = 3 * K - 1
        W1 = (rng.standard_normal((H, D - n1)) * 0.8 / np.sqrt(D - n1)).astype(f32)
        c1 = (rng.standard_normal(H) * 0.3).astype(f32)
        W2 = (rng.standard_normal((J * n1, H)) * 0.3 / np.sqrt(H)).astype(f32)
        c2 = (rng.standard_normal(J * n1) * 0.3).astype(f32)
        dev.append(B.Coupling(B.MLPSplineConditioner(W1, c1, W2, c2, K=K, B=Bv, activation="tanh"),
                              B.PartitionMask(D, idx1, idx2)))
        ora.append(C.MLPSplineLayer(idx1, idx2, W1, c1, W2, c2, K, Bv, "tanh"))
    return B.Composed(*dev), ora


def test_spline_chain_logpdf_and_vjp(B):
    import torch

    rng = np.random.default_rng(31)
    D, N = 32, 4000
    flow, ora = _spline_flow(B, rng, D)
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.3, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu=mu, sigma=sigma), flow)
    y = (rng.standard_normal((D, N)) * 0.8).astype(f32)
    yd = B.from_numpy(y)
    lp = B.to_numpy(B.logpdf(td, yd))
    inv_layers, flags = ora[::-1], [True] * len(ora)
    lb = rng.standard_normal(N)
    g, grads, base = E.chain_vjp(inv_layers, flags, y.astype(np.float64), None, lb, mu, sigma, terminal=True)
    ybar, fgrads, bgrads = B.logpdf_vjp(td, yd, torch.from_numpy(lb.astype(f32)).cuda())
    assert rel(B.to_numpy(ybar), g) < 1e-4
    flow_grads = grads[::-1]
    for k in (0, 2):
        assert rel(fgrads[k]["factors"].cpu().numpy(), flow_grads[k]["factors"]) < 2e-4, k
    assert rel(bgrads["σ"].cpu().numpy(), base["σ"]) < 1e-4
    # the logpdf itself against the float64 chain
    cur, lj = y.astype(np.float64), np.zeros(N)
    for lay in inv_layers:
        cur, l = lay.inverse(cur)
        lj += l
    lp64 = O.mvnormal_diag_logpdf(mu, sigma, cur) + lj
    assert rel(lp, lp64) < 1e-5
    # chain_vjp through the forward flow
    x = (rng.standard_normal((D, N)) * 0.8).astype(f32)
    yb = rng.standard_normal((D, N))
    xbar, cg = B.chain_vjp(flow, B.from_numpy(x), B.from_numpy(yb.astype(f32)))
    g2, grads2 = E.chain_vjp(ora, [False] * len(ora), x.astype(np.float64), yb, None)[:2]
    assert rel(B.to_numpy(xbar), g2) < 1e-4
    for k in (0, 2):
        assert rel(cg[k]["factors"].cpu().numpy(), grads2[k]["factors"]) < 2e-4, k


def test_rand_logpdf_and_rand_vjp_through_the_layer(B):
    import torch

    rng = np.random.default_rng(41)
    D, N, SEED = 48, 6000, 1234
    F, dst, p = lu_params(rng, D, "random")
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.3, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu=mu, sigma=sigma), B.LULinear(F, p))
    z = O.philox_normals(SEED, 0, D, N)
    x = B.to_numpy(B.rand(td.dist, N, seed=SEED))
    y, lq = B.rand_logpdf(td, N, seed=SEED)
    y64, lj64 = S.forward(F, dst, x.astype(np.float64))
    assert rel(B.to_numpy(y), y64) < 1e-5
    lq64 = O.mvnormal_diag_logpdf(mu, sigma, x.astype(np.float64)) - lj64
    assert rel(B.to_numpy(lq), lq64) < 1e-5
    ybar = torch.from_numpy(rng.standard_normal((D, N)).astype(f32)).cuda()
    qbar = torch.from_numpy(rng.standard_normal(N).astype(f32)).cuda()
    fg, bg = B.rand_vjp(td, N, B.from_numpy(ybar.cpu().numpy()), qbar, seed=SEED)
    g64, b64 = R.vjp([S.LULayer(F, dst)], [False], z, ybar.cpu().numpy(), qbar.cpu().numpy(), mu, sigma, x=x)
    assert rel(fg[0]["factors"].cpu().numpy(), g64[0]["factors"]) < 2e-4
    assert rel(bg["μ"].cpu().numpy(), b64["μ"]) < 2e-4 and rel(bg["σ"].cpu().numpy(), b64["σ"]) < 2e-4


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,N", [(5, 300), (64, 200), (300, 100), (2048, 24)])
def test_float64(B, D, N, inv):
    import torch

    rng = np.random.default_rng(D + 2 * inv)
    F = S.random_lu(rng, D, np.float64)
    dst = rng.permutation(D)
    x, ybar, lbar = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    lay = B.LULinear(F, dst + 1, dtype=torch.float64)
    t = B.inverse(lay) if inv else lay
    xd = B.from_numpy(x, dtype=np.float64)
    y, lj = B.with_logabsdet_jacobian(t, xd)
    y64, l64 = (S.inverse if inv else S.forward)(F, dst, x)
    assert rel(B.to_numpy(y), y64) < 1e-12 and np.abs(B.to_numpy(lj) - l64).max() <= 1e-12 * max(1.0, abs(l64[0]))
    xbar, grads = B.chain_vjp(t, xd, B.from_numpy(ybar, dtype=np.float64), torch.from_numpy(lbar).cuda())
    xb64, Fb64 = S.vjp(F, dst, x, ybar, lbar, inverse=inv)
    assert rel(B.to_numpy(xbar), xb64) < 1e-12 and rel(grads[0]["factors"].cpu().numpy(), Fb64) < 1e-11
    # the same chain with a triangular layer in it runs the Float64 kernels holding both cases
    tc = B.Composed(t, B.Scale(B.UpperTriangular(F), dtype=torch.float64))
    yc, _ = B.with_logabsdet_jacobian(tc, xd)
    assert rel(B.to_numpy(yc), T.view(F, True, False) @ y64) < 1e-12


def test_flow_training(B):
    """autograd.Flow(Coupling(MLPSplineConditioner) ∘ LULinear ∘ Coupling ∘ LULinear, MvNormal(D)): the first gradient
    of the NLL matches the float64 oracle, and Adam lowers the NLL."""
    import torch

    rng = np.random.default_rng(81)
    D, N = 16, 8192
    flow_t, ora = _spline_flow(B, rng, D)
    flow = B.autograd.Flow(flow_t, B.MvNormal(D))
    Q, _ = np.linalg.qr(rng.standard_normal((D, D)))
    data = (Q @ np.diag(np.linspace(0.5, 1.5, D)) @ rng.standard_normal((D, N))).astype(f32)
    y = B.from_numpy(data)
    Fs = [lay._F for lay in B.flatten(flow_t) if isinstance(lay, B.LULinear)]
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    opt.zero_grad()
    nll0 = flow.nll(y)
    nll0.backward()
    _, grads, _ = E.chain_vjp(ora[::-1], [True] * len(ora), data.astype(np.float64), None, -np.ones(N), None, None,
                              terminal=True)
    flow_grads = grads[::-1]
    params = {p.data_ptr(): p for p in flow.params}
    for F_dev, k in zip(Fs, (0, 2)):
        g = params[F_dev.data_ptr()].grad.t().cpu().numpy()  # storage is Fᵀ row-major
        assert rel(g, flow_grads[k]["factors"]) < 2e-4, k
    opt.step()
    losses = [float(nll0.detach())]
    for _ in range(30):
        opt.zero_grad()
        loss = flow.nll(y)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0] - 0.01 * abs(losses[0]), losses[::10]
