"""GPU tests of the dense Scale layer, B2B_SCALE_MATRIX: Scale(A) with a D x D matrix, against the float64 restatement of
tests/scale_matrix_oracle.py.  y is held to a componentwise GEMM bound, (4·D + 2)·eps32·(|M||x|) with M = A (forward) or
A⁻¹ (inverse, times the asserted condition number of A), and log|det A| to about 1e-6·D."""
import ctypes

import numpy as np
import pytest

import chain_vjp_oracle as V
import mvnormal_tril_oracle as T
import scale_matrix_oracle as S
import spline_coupling_oracle as SC
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


def stream():
    from bijectors_jl_b200.interface import _stream

    return _stream()


def matrix(rng, D, kind):
    """float32 A: well conditioned (I + 0.3·G/√D), with A₁₁ = 0 (the first step must pivot), or with det A < 0."""
    A = S.well_conditioned(rng, D)
    if kind == "pivot" and D >= 2:
        A[[0, 1]] = A[[1, 0]]
        A[0, 0] = 0.0
    if kind == "negdet":
        A[:, 0] = -A[:, 0]
    A = A.astype(f32)
    if D >= 2:
        assert np.linalg.cond(A.astype(np.float64)) < COND_MAX
    if kind == "negdet":
        assert np.linalg.det(A.astype(np.float64)) < 0
    return A


def check_y(y, A, x, inv):
    A64, x64 = A.astype(np.float64), x.astype(np.float64)
    M = np.linalg.inv(A64) if inv else A64
    y64 = M @ x64
    bound = (4 * A.shape[0] + 2) * EPS * (np.abs(M) @ np.abs(x64)) * (COND_MAX if inv else 1.0) + 1e-30
    err = np.abs(np.asarray(y, np.float64) - y64)
    assert (err <= bound).all(), float((err / bound).max())


def check_lj(lj, A, inv, acc=None):
    ld = S.logabsdet(A) * (-1 if inv else 1)
    want = ld if acc is None else acc.astype(np.float64) + ld
    assert np.abs(np.asarray(lj, np.float64) - want).max() <= 1e-6 * A.shape[0] + 2e-7 * np.abs(want).max() + 1e-6


SHAPES = [(1, 1), (2, 0), (3, 1001), (17, 129), (32, 1000), (64, (1 << 19) + 3), (100, 333), (128, 4099), (255, 257),
          (256, 1000)]


@pytest.mark.parametrize("kind", ["plain", "pivot", "negdet"])
@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,N", SHAPES)
def test_parity(B, D, N, inv, kind):
    rng = np.random.default_rng(D * 13 + N % 1000 + 7 * inv + len(kind))
    A = matrix(rng, D, kind)
    x = rng.standard_normal((D, N)).astype(f32)
    lay = B.Scale(A)
    xd = B.from_numpy(x) if N else B.colmajor_empty(D, 0, "cuda")
    y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, xd)
    assert tuple(y.shape) == (D, N) and tuple(lj.shape) == (N,)
    if N == 0:
        return
    y, lj = B.to_numpy(y), B.to_numpy(lj)
    check_y(y, A, x, inv)
    check_lj(lj, A, inv)


def _raw(B, lay, inv, D, N, x, ldx, xoff, y, ldy, yoff, lj, acc):
    import torch

    from bijectors_jl_b200.interface import _desc_array

    arr = _desc_array(lay._descs(inv, D))
    L = B.lib()
    wsb = L.b2b_chain_workspace_bytes(arr, 1, D, N, 1 if y is not None else 0, 0)
    assert wsb > 0
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    p = lambda t, off: None if t is None else t.data_ptr() + 4 * off  # noqa: E731
    rc = L.b2b_chain_run_f32(arr, 1, p(x, xoff), p(y, yoff), p(lj, 0), None, D, N, ldx, ldy, acc, ws.data_ptr(), wsb,
                             stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D", [5, 130])
def test_call_modes(B, D, inv):
    """Padded ld and misaligned bases, accumulate, y == NULL and in place give the bits of the plain call."""
    import torch

    rng = np.random.default_rng(11 + inv + D)
    N = 333
    A = matrix(rng, D, "plain")
    x = rng.standard_normal((D, N)).astype(f32)
    lay = B.Scale(A)
    t = B.inverse(lay) if inv else lay
    y0, l0 = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(t, B.from_numpy(x)))
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


def test_round_trip(B):
    rng = np.random.default_rng(3)
    D, N = 96, 5000
    A = matrix(rng, D, "pivot")
    x = rng.standard_normal((D, N)).astype(f32)
    lay = B.Scale(A)
    y, lj = B.with_logabsdet_jacobian(lay, B.from_numpy(x))
    xr, ljr = B.with_logabsdet_jacobian(B.inverse(lay), y)
    assert rel(B.to_numpy(xr), x) < 1e-5
    assert B.to_numpy(ljr).tobytes() == (-B.to_numpy(lj)).tobytes()


def test_singular_forward(B):
    rng = np.random.default_rng(4)
    D, N = 40, 700
    A = matrix(rng, D, "plain")
    A[:, 7] = 0.0
    x = rng.standard_normal((D, N)).astype(f32)
    y, lj = B.with_logabsdet_jacobian(B.Scale(A), B.from_numpy(x))
    check_y(B.to_numpy(y), A, x, False)
    assert (B.to_numpy(lj) == -np.inf).all()


def _chain(B, rng, D):
    """Scale ∘ spline coupling ∘ BatchNorm ∘ Permute ∘ Scale ∘ affine coupling ∘ RQS ∘ Planar, device and oracle layers."""
    dev, ora = [], []
    w, u = (rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32)
    bb = rng.standard_normal(1).astype(f32)
    dev.append(B.PlanarLayer(w, u, bb))
    ora.append(O.Layer("planar", dict(w=w, u=u, b=bb)))
    K = 8
    spl = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                    rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    Wk, Hk, Dk = spl.knots()
    dev.append(spl)
    ora.append(O.Layer("rqs", dict(widths=Wk, heights=Hk, derivs=Dk)))
    n1 = D // 2
    cW = (rng.standard_normal((2 * n1, D - n1)) * 0.05).astype(f32)
    cc = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    i1, i2 = list(range(1, n1 + 1)), list(range(n1 + 1, D + 1))
    dev.append(B.Coupling(B.AffineConditioner(cW, cc), B.PartitionMask(D, i1, i2)))
    ora.append(O.Layer("coupling_affine", dict(idx1=np.asarray(i1), idx2=np.asarray(i2), W=cW, c=cc)))
    A1 = matrix(rng, D, "negdet")
    dev.append(B.Scale(A1))
    ora.append(S.ScaleLayer(A1))
    perm = rng.permutation(D) + 1
    dev.append(B.Permute(perm))
    ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))))
    b, logs = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
    m, v = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    dev.append(B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v))
    ora.append(O.Layer("batchnorm", dict(bn=O.BatchNormParams(b=b, logs=logs, m=m, v=v, eps=1e-5))))
    si1, si2, sW, sc = list(range(2, D + 1, 2)), list(range(1, D + 1, 2)), None, None
    sW = (rng.standard_normal(((3 * 6 - 1) * len(si1), len(si2))) * 0.3 / np.sqrt(len(si2))).astype(f32)
    sc = (rng.standard_normal((3 * 6 - 1) * len(si1)) * 0.3).astype(f32)
    dev.append(B.Coupling(B.SplineConditioner(sW, sc, K=6, B=3.0), B.PartitionMask(D, si1, si2)))
    ora.append(SC.SplineLayer(si1, si2, sW, sc, 6, 3.0))
    A2 = matrix(rng, D, "pivot")
    dev.append(B.Scale(A2))
    ora.append(S.ScaleLayer(A2))
    return B.Composed(*dev), ora


def test_chain_forward_inverse(B):
    rng = np.random.default_rng(21)
    D, N = 16, 900
    flow, ora = _chain(B, rng, D)
    x = (rng.standard_normal((D, N)) * 0.8).astype(f32)
    y, lj = B.with_logabsdet_jacobian(flow, B.from_numpy(x))
    y64, l64 = O.chain_forward(ora, x.astype(np.float64))
    assert rel(B.to_numpy(y), y64) < 1e-5 and rel(B.to_numpy(lj), l64) < 1e-5
    xr, ljr = B.with_logabsdet_jacobian(B.inverse(flow), y)
    x64, li64 = O.chain_inverse(ora, y64)
    assert rel(B.to_numpy(xr), x64) < 1e-4 and rel(B.to_numpy(ljr), li64) < 1e-4


@pytest.mark.parametrize("base", ["diag", "tril"])
def test_logpdf_and_chain_vjp(B, base):
    import torch

    rng = np.random.default_rng(31 + (base == "tril"))
    D, N = 16, 800
    flow, ora = _chain(B, rng, D)
    y = (rng.standard_normal((D, N)) * 0.8).astype(f32)
    mu = (rng.standard_normal(D) * 0.2).astype(f32)
    if base == "diag":
        sigma = rng.uniform(0.7, 1.3, D).astype(f32)
        dist = B.MvNormal(D, mu=mu, sigma=sigma)
    else:
        L = T.random_tril(rng, D).astype(f32)
        dist = B.MvNormal(D, mu=mu, scale_tril=L)
    td = B.transformed(dist, flow)
    yd = B.from_numpy(y)
    lp = B.to_numpy(B.logpdf(td, yd))
    inv_layers = ora[::-1]
    cur, lj = y.astype(np.float64), 0.0
    for lay in inv_layers:
        cur, l = lay.inverse(cur)
        lj = lj + l
    if base == "diag":
        lp64 = O.mvnormal_diag_logpdf(mu.astype(np.float64), sigma.astype(np.float64), cur) + lj
    else:
        lp64 = T.logpdf(L, mu, cur, np.float64) + lj
    assert rel(lp, lp64) < 1e-5
    s, lps = B.logpdf_sum(td, yd)
    assert B.to_numpy(lps).tobytes() == lp.tobytes()
    assert abs(float(s) - lp64.sum()) <= 1e-5 * abs(lp64.sum())
    lb = rng.standard_normal(N)
    ybar, fgrads, _ = B.logpdf_vjp(td, yd, torch.from_numpy(lb.astype(f32)).cuda())
    flags = [True] * len(inv_layers)
    if base == "diag":
        g, grads, _ = V.chain_vjp(inv_layers, flags, y, None, lb, mu, sigma, terminal=True)
    else:
        g, grads, _ = V.chain_vjp(inv_layers, flags, y, None, lb, mu, scale_tril=L)
    assert rel(B.to_numpy(ybar), g) < 1e-3
    flow_grads = grads[::-1]
    for k in (3, 7):
        assert rel(fgrads[k]["a"].cpu().numpy(), flow_grads[k]["a"]) < 1e-3, k


@pytest.mark.parametrize("ljb", [False, True])
@pytest.mark.parametrize("yb", [False, True])
@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,N", [(1, 50), (3, 1001), (64, 20000), (200, 3000), (256, 1500)])
def test_vjp(B, D, N, inv, yb, ljb):
    import torch

    rng = np.random.default_rng(D + N + 2 * inv + 4 * yb + 8 * ljb)
    A = matrix(rng, D, "pivot")
    x = rng.standard_normal((D, N)).astype(f32)
    ybar = rng.standard_normal((D, N)).astype(f32) if yb else None
    lbar = rng.standard_normal(N).astype(f32) if ljb else None
    lay = B.Scale(A)
    t = B.inverse(lay) if inv else lay
    xbar, grads = B.chain_vjp(t, B.from_numpy(x), None if ybar is None else B.from_numpy(ybar),
                              None if lbar is None else torch.from_numpy(lbar).cuda())
    xb64, Ab64 = S.vjp(A, x, ybar, lbar, inverse=inv)
    xb = B.to_numpy(xbar)
    if yb:
        check_y(xb, A.T.copy(), ybar, inv)
    else:
        assert not xb.any()
    Ab = grads[0]["a"].cpu().numpy()
    if yb or ljb:
        assert rel(Ab, Ab64) < 2e-4, rel(Ab, Ab64)
    else:
        assert not Ab.any()


def test_repeatable_and_graph_replay(B):
    import torch

    rng = np.random.default_rng(61)
    D, N = 128, 20000
    flow, _ = _chain(B, rng, D)
    x = B.from_numpy((rng.standard_normal((D, N)) * 0.8).astype(f32))
    yb = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lb = torch.randn(N, device="cuda")
    r1 = B.with_logabsdet_jacobian(flow, x)
    r2 = B.with_logabsdet_jacobian(flow, x)
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[1], r2[1])
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


def test_rand_and_host_path(B):
    import torch

    rng = np.random.default_rng(41)
    D, N = 256, 3001
    A = matrix(rng, D, "negdet")
    lay = B.Scale(A)
    td = B.transformed(B.MvNormal(D), lay)
    y, lj = B.rand(td, N, seed=77, offset=2, with_logjac=True)
    z = O.philox_normals(77, 2, D, N)
    check_y(B.to_numpy(y), A, z.astype(f32), False)
    check_lj(B.to_numpy(lj), A, False)
    x = B.rand(td.dist, N, seed=77, offset=2)
    y2, lj2 = B.run_chain(lay, x)
    assert B.to_numpy(y).tobytes() == B.to_numpy(y2).tobytes() and B.to_numpy(lj).tobytes() == B.to_numpy(lj2).tobytes()
    xh = B.from_numpy(B.to_numpy(x), device="cpu")
    yh, ljh = B.run_chain(lay, xh)
    assert B.to_numpy(yh).tobytes() == B.to_numpy(y2).tobytes()
    assert B.to_numpy(ljh).tobytes() == B.to_numpy(lj2).tobytes()
    xr, _ = B.run_chain(B.inverse(lay), xh)
    xr_dev, _ = B.run_chain(B.inverse(lay), x)
    assert B.to_numpy(xr).tobytes() == B.to_numpy(xr_dev).tobytes()
    # a full-covariance base through the TRIL sampler
    Lt = T.random_tril(rng, D).astype(f32)
    td2 = B.transformed(B.MvNormal(D, scale_tril=Lt), lay)
    y3 = B.to_numpy(B.rand(td2, 500, seed=5))
    base = B.to_numpy(B.rand(td2.dist, 500, seed=5))
    check_y(y3, A, base, False)
    del torch


def _desc(B, D, inverse=0, dtype=None):
    import torch

    A = torch.eye(max(D, 1), device="cuda", dtype=dtype or torch.float32)
    d = B._lib.LayerDesc64() if dtype is not None else B._lib.LayerDesc()
    d.kind, d.inverse, d.p0 = B._lib.SCALE_MATRIX, inverse, A.data_ptr()
    return d, A


def test_slot_status_codes(B):
    import torch

    L = B.lib()
    D, N = 8, 64
    x = torch.zeros((N * D,), device="cuda")
    xb = torch.zeros((N * D,), device="cuda")
    for slot, want in [(1, -2), (2, -2), (3, -2), (0, 0)]:
        d, keep = _desc(B, D)
        arr = (B._lib.LayerDesc * 1)(d)
        bar = torch.zeros((D * D,), device="cuda")
        ptrs = (ctypes.c_void_p * 4)()
        ptrs[slot] = bar.data_ptr()
        wsb = L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
        ws = torch.empty((wsb,), dtype=torch.uint8, device="cuda")
        rc = L.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(ptrs, ctypes.c_void_p), D, N, D,
                                 D, D, ws.data_ptr(), wsb, stream())
        assert rc == want, (slot, rc)
    torch.cuda.synchronize()


@pytest.mark.parametrize("inv", [0, 1])
def test_past_the_envelope(B, inv):
    import torch

    L = B.lib()
    D, N = 257, 100
    d, keep = _desc(B, D, inv)
    arr = (B._lib.LayerDesc * 1)(d)
    x = torch.zeros((N * D,), device="cuda")
    y = torch.full((N * D,), 3.5, device="cuda")
    lj = torch.full((N,), 3.5, device="cuda")
    xb = torch.full((N * D,), 3.5, device="cuda")
    torch.cuda.synchronize()
    assert L.b2b_chain_workspace_bytes(arr, 1, D, N, 1, 0) == 0 and L.b2b_workspace_bytes(arr, D, N) == 0
    assert L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N) == 0
    assert L.b2b_chain_run_f32(arr, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream()) == -2
    assert L.b2b_last_launch_count() == 0
    assert L.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, None, 0, stream()) == -2
    assert L.b2b_last_launch_count() == 0
    torch.cuda.synchronize()
    assert (y == 3.5).all() and (lj == 3.5).all() and (xb == 3.5).all()
    # inside the envelope the call without workspace asks for it, with nothing launched
    d2, keep2 = _desc(B, 8, inv)
    arr2 = (B._lib.LayerDesc * 1)(d2)
    assert L.b2b_chain_workspace_bytes(arr2, 1, 8, N, 1, 0) > 12 * 64
    assert L.b2b_chain_run_f32(arr2, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, 8, N, 8, 8, 0, None, 0, stream()) == -3
    assert L.b2b_last_launch_count() == 0


def test_float64_descriptor_unsupported(B):
    import torch

    L = B.lib()
    D, N = 8, 16
    d, keep = _desc(B, D, 0, torch.float64)
    arr = (B._lib.LayerDesc64 * 1)(d)
    x = torch.zeros(D * N, dtype=torch.float64, device="cuda")
    y = torch.zeros(D * N, dtype=torch.float64, device="cuda")
    assert L.b2b_chain_run_f64(arr, 1, x.data_ptr(), y.data_ptr(), None, None, D, N, D, D, 0, None, 0, stream()) == -2
    assert L.b2b_chain_vjp_workspace_bytes_f64(arr, 1, D, N) == 0
    assert L.b2b_chain_vjp_f64(arr, 1, x.data_ptr(), None, None, y.data_ptr(), None, D, N, D, D, D, None, 0, stream()) == -2


def test_training_lowers_nll_and_first_gradient(B):
    """Flow(Scale(A) ∘ RationalQuadraticSpline) over an MvNormal base: the first gradient of A matches the float64 oracle
    and a few Adam steps lower the NLL."""
    import torch

    rng = np.random.default_rng(81)
    D, N, K = 6, 4096, 8
    A = matrix(rng, D, "plain")
    wr, hr, dr = (rng.standard_normal((D, K)) * 0.1).astype(f32), (rng.standard_normal((D, K)) * 0.1).astype(f32), \
        (rng.standard_normal((D, K - 1)) * 0.1).astype(f32)
    spl = B.RationalQuadraticSpline(wr, hr, dr, 4.0)
    Wk, Hk, Dk = spl.knots()
    sc = B.Scale(A)
    flow = B.autograd.Flow(B.Composed(spl, sc), B.MvNormal(D))
    mix = np.linalg.qr(rng.standard_normal((D, D)))[0] * np.linspace(0.3, 2.0, D)
    data = (mix @ rng.standard_normal((D, N))).astype(f32)
    y = B.from_numpy(data)
    nll = flow.nll(y)
    nll.backward()
    # oracle: logpdf(y) = logpdf_base(spl⁻¹(A⁻¹ y)) + log|det A⁻¹| + spline inverse log-Jacobian
    sl, scl = O.Layer("rqs", dict(widths=Wk, heights=Hk, derivs=Dk)), S.ScaleLayer(A)
    u0 = data.astype(np.float64)
    u1, l1 = scl.inverse(u0)
    u2, l2 = sl.inverse(u1)
    lp = O.mvnormal_diag_logpdf(None, None, u2) + l1 + l2
    assert abs(float(nll) + lp.sum()) <= 1e-4 * abs(lp.sum())
    g = V.mvnormal_diag_logpdf_vjp(np.zeros(D), np.ones(D), u2, -np.ones(N))[0]
    g, _ = V._layer_vjp(sl, True, u1, g, -np.ones(N))
    _, ga = scl.vjp(u0, g, -np.ones(N), inverse=True)
    p = [q for q in flow.params if q.shape == (D, D)][0]
    assert rel(p.grad.cpu().numpy().T, ga["a"]) < 1e-3
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    first = float(nll)
    for _ in range(30):
        opt.zero_grad()
        loss = flow.nll(y)
        loss.backward()
        opt.step()
    assert float(flow.nll(y)) < first - 0.02 * abs(first)
