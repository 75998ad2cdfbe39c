"""GPU tests of the spline coupling layer, B2B_COUPLING_RQS: Coupling(x₂ -> RationalQuadraticSpline(…, B), mask) against
the float64 reference of tests/spline_coupling_oracle.py.  Gates are tied to the reference's own float32 error on the same
input, as in test_gpu_parity.gate: max(1e-5, 2 × ‖oracle32 − oracle64‖ / ‖oracle64‖), norm-wise."""
import ctypes

import numpy as np
import pytest

import chain_vjp_oracle as V
import mvnormal_tril_oracle as T
import spline_coupling_oracle as S
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(dev, a64, a32, what=""):
    tol = max(RTOL, 2.0 * rel(a32, a64))
    e = rel(dev, a64)
    assert e <= tol, (what, e, tol)


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def spec(rng, D, n1, n2, K, scattered=False, with_c=True, scale=0.6):
    rows = (rng.permutation(D) if scattered else np.arange(D)) + 1
    idx1, idx2 = [int(i) for i in rows[:n1]], [int(i) for i in rows[n1:n1 + n2]]
    J = 3 * K - 1
    Wm = (rng.standard_normal((J * n1, n2)) * scale / np.sqrt(n2)).astype(f32)
    c = (rng.standard_normal(J * n1) * 0.5).astype(f32) if with_c else None
    return idx1, idx2, Wm, c


def batch(rng, D, N, Bv):
    """Uniform on [−B/0.95, B/0.95]: about 5 % of the elements lie outside the box."""
    return rng.uniform(-Bv / 0.95, Bv / 0.95, (D, N)).astype(f32)


def layer(B, D, idx1, idx2, Wm, c, K, Bv):
    return B.Coupling(B.SplineConditioner(Wm, c, K=K, B=Bv), B.PartitionMask(D, idx1, idx2))


def stream():
    from bijectors_jl_b200.interface import _stream

    return _stream()


def ptr(t, off=0):
    return None if t is None else t.data_ptr() + 4 * off


# D, n1, n2, K, N, scattered (x₃ rows exist whenever n1 + n2 < D)
SHAPES = [
    (2, 1, 1, 2, 17, False),
    (3, 1, 1, 5, 1000, True),
    (10, 4, 5, 8, 1000, True),
    (10, 5, 5, 8, 1, False),
    (32, 16, 16, 16, 1000, False),
    (64, 32, 32, 8, 65539, False),
    (128, 64, 64, 5, 1000, True),
    (200, 100, 90, 8, 17, True),
    (256, 128, 128, 8, 1000, False),
    (1000, 1, 128, 16, 17, True),
    (1000, 128, 100, 2, 1000, True),
]


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,n1,n2,K,N,scattered", SHAPES)
def test_parity(B, D, n1, n2, K, N, scattered, inv):
    rng = np.random.default_rng(D * 7 + n1 + K + N + inv)
    Bv = 3.0
    idx1, idx2, Wm, c = spec(rng, D, n1, n2, K, scattered)
    x = batch(rng, D, N, Bv)
    lay = layer(B, D, idx1, idx2, Wm, c, K, Bv)
    y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, B.from_numpy(x))
    y, lj = B.to_numpy(y), B.to_numpy(lj)
    f = S.inverse if inv else S.forward
    cols = None if N <= 1000 else np.unique(np.r_[0, 1, N - 1, rng.integers(0, N, 300)])
    y64, l64 = f(idx1, idx2, Wm, c, K, Bv, x.astype(np.float64), np.float64, cols)
    y32, l32 = f(idx1, idx2, Wm, c, K, Bv, x, f32, cols)
    sel = slice(None) if cols is None else cols
    r1 = np.asarray(idx1) - 1
    gate(y[r1][:, sel], y64[r1], y32[r1], "y1")
    gate(lj[sel], l64, l32, "logjac")
    rest = np.setdiff1d(np.arange(D), r1)
    assert y[rest].tobytes() == x[rest].tobytes()  # x₂ and x₃ bit-exact, whole batch
    assert np.isfinite(y).all() and np.isfinite(lj).all()


def test_inverse_of_forward(B):
    rng = np.random.default_rng(3)
    D, N, K, Bv = 48, 2000, 8, 2.5
    idx1, idx2, Wm, c = spec(rng, D, 20, 24, K, scattered=True)
    x = batch(rng, D, N, Bv)
    lay = layer(B, D, idx1, idx2, Wm, c, K, Bv)
    y, lj = B.with_logabsdet_jacobian(lay, B.from_numpy(x))
    xr, ljr = B.with_logabsdet_jacobian(B.inverse(lay), y)
    assert rel(B.to_numpy(xr), x) < 5e-5  # a float32 round trip through the spline and its inverse
    assert rel(B.to_numpy(ljr), -B.to_numpy(lj)) < 1e-4


def _raw(B, lay, inv, D, N, x, ldx, xoff, y, ldy, yoff, lj, acc):
    import torch

    from bijectors_jl_b200.interface import _desc_array

    arr = _desc_array(lay._descs(inv, D))
    L = B.lib()
    wsb = L.b2b_chain_workspace_bytes(arr, 1, D, N, 1 if y is not None else 0, 0)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device="cuda")
    rc = L.b2b_chain_run_f32(arr, 1, ptr(x, xoff), ptr(y, yoff), ptr(lj), None, D, N, ldx, ldy, acc, ws.data_ptr(), wsb,
                             stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("inv", [False, True])
def test_layouts(B, inv):
    """Padded ld, misaligned bases, in place, accumulate and logjac only give the bits of the plain call."""
    import torch

    rng = np.random.default_rng(11 + inv)
    D, N, K, Bv = 10, 333, 5, 2.0
    idx1, idx2, Wm, c = spec(rng, D, 4, 3, K, scattered=True)
    x = batch(rng, D, N, Bv)
    lay = layer(B, D, idx1, idx2, Wm, c, K, Bv)
    t = B.inverse(lay) if inv else lay
    y0, l0 = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(t, B.from_numpy(x)))
    ld = D + 3
    sentinel = 7.25
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
    # accumulate
    base = torch.randn(N, device="cuda")
    lj.copy_(base)
    assert _raw(B, lay, inv, D, N, xb, ld, 1, yb, ld, 3, lj, 1) == 0
    assert lj.cpu().numpy().tobytes() == (base.cpu().numpy() + l0).astype(f32).tobytes()
    # logjac only
    lj.fill_(0)
    assert _raw(B, lay, inv, D, N, xb, ld, 1, None, D, 0, lj, 0) == 0
    assert lj.cpu().numpy().tobytes() == l0.tobytes()
    # in place
    assert _raw(B, lay, inv, D, N, xb, ld, 1, xb, ld, 1, lj, 0) == 0
    assert xv[:, :D].cpu().numpy().T.tobytes() == y0.tobytes()
    assert (xv[:, D:] == sentinel).all() and lj.cpu().numpy().tobytes() == l0.tobytes()


def test_zero_W_is_the_plain_spline(B):
    """With W = 0 every column gets the knots of c: the x₁ rows equal RationalQuadraticSpline(reshape(c…), B) run through
    the existing RQS path."""
    rng = np.random.default_rng(5)
    D, N, K, Bv, n1 = 12, 4000, 8, 2.0, 7
    idx1, idx2, _, c = spec(rng, D, n1, 5, K)
    Wm = np.zeros(((3 * K - 1) * n1, 5), f32)
    x = batch(rng, D, N, Bv)
    y, lj = B.with_logabsdet_jacobian(layer(B, D, idx1, idx2, Wm, c, K, Bv), B.from_numpy(x))
    rw, rh, rd = S.raw_params(Wm, c, np.zeros(5, f32), K, f32)
    rqs = B.RationalQuadraticSpline(rw, rh, rd, Bv)
    x1 = np.ascontiguousarray(x[:n1])
    ys, ljs = B.with_logabsdet_jacobian(rqs, B.from_numpy(x1))
    y64, l64 = O.rqs_forward(*O.rqs_params(*(a.astype(np.float64) for a in (rw, rh, rd)), Bv), x1.astype(np.float64))
    y32, l32 = O.rqs_forward(*O.rqs_params(rw, rh, rd, Bv), x1)
    tol_y = max(RTOL, 2 * rel(y32, y64))
    tol_l = max(RTOL, 2 * rel(l32, l64))
    assert rel(B.to_numpy(y)[:n1], B.to_numpy(ys)) <= tol_y
    assert rel(B.to_numpy(lj), B.to_numpy(ljs)) <= tol_l


def _flow(B, rng, D, K=6, Bv=3.0):
    """Planar ∘ Permute ∘ spline coupling ∘ BatchNorm ∘ spline coupling, device and oracle layers."""
    dev, ora = [], []
    i1, i2, W1, c1 = spec(rng, D, D // 2, D - D // 2, K)
    dev.append(layer(B, D, i1, i2, W1, c1, K, Bv))
    ora.append(S.SplineLayer(i1, i2, W1, c1, K, Bv))
    b, logs = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
    m, v = (rng.standard_normal(D) * 0.1).astype(f32), (rng.uniform(0.5, 1.5, D)).astype(f32)
    dev.append(B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v))
    ora.append(O.Layer("batchnorm", dict(bn=O.BatchNormParams(b=b, logs=logs, m=m, v=v, eps=1e-5))))
    perm = rng.permutation(D) + 1
    dev.append(B.Permute(perm))
    ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))))
    i1, i2, W2, c2 = spec(rng, D, D // 3, D - D // 3 - 1, K, scattered=True)
    dev.append(layer(B, D, i1, i2, W2, c2, K, Bv))
    ora.append(S.SplineLayer(i1, i2, W2, c2, K, Bv))
    w, u = (rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32)
    bb = rng.standard_normal(1).astype(f32)
    dev.append(B.PlanarLayer(w, u, bb))
    ora.append(O.Layer("planar", dict(w=w, u=u, b=bb)))
    return B.Composed(*dev), ora


def test_chain_forward_inverse(B):
    rng = np.random.default_rng(21)
    D, N = 16, 700
    flow, ora = _flow(B, rng, D)
    x = batch(rng, D, N, 2.0)
    y, lj = B.with_logabsdet_jacobian(flow, B.from_numpy(x))
    y64, l64 = O.chain_forward(ora, x.astype(np.float64))
    y32, l32 = O.chain_forward(ora, x)
    gate(B.to_numpy(y), y64, y32, "y")
    gate(B.to_numpy(lj), l64, l32, "logjac")
    xr, ljr = B.with_logabsdet_jacobian(B.inverse(flow), y)
    x64, li64 = O.chain_inverse(ora, y64)
    x32, li32 = O.chain_inverse(ora, y32)
    gate(B.to_numpy(xr), x64, x32, "x")
    gate(B.to_numpy(ljr), li64, li32, "inverse logjac")


@pytest.mark.parametrize("base", ["diag", "tril"])
def test_logpdf_and_vjp(B, base):
    import torch

    rng = np.random.default_rng(31 + (base == "tril"))
    D, N = 16, 600
    flow, ora = _flow(B, rng, D)
    y = batch(rng, D, N, 2.0)
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
    inv_layers, flags = ora[::-1], [True] * len(ora)

    def chain_lp(yy, dt):
        cur, lj = np.asarray(yy, dt), 0.0
        for lay in inv_layers:
            cur, l = lay.inverse(cur)
            lj = lj + l
        if base == "diag":
            return O.mvnormal_diag_logpdf(mu.astype(dt), sigma.astype(dt), cur) + lj, cur
        return T.logpdf(L, mu, cur, dt) + lj, cur

    lp64, x64 = chain_lp(y, np.float64)
    lp32, _ = chain_lp(y, f32)
    gate(lp, lp64, lp32, "logpdf")
    s, lps = B.logpdf_sum(td, yd)
    assert B.to_numpy(lps).tobytes() == lp.tobytes()
    assert abs(float(s) - lp64.sum()) <= max(1e-5, 2 * abs(lp32.sum(dtype=np.float64) - lp64.sum())) * abs(lp64.sum()) + 1e-3
    # reverse mode: ȳ and the W̄ / c̄ of both spline layers
    lb = rng.standard_normal(N)
    ybar, fgrads, _ = B.logpdf_vjp(td, yd, torch.from_numpy(lb.astype(f32)).cuda())
    if base == "diag":
        g, grads, _ = V.chain_vjp(inv_layers, flags, y, None, lb, mu, sigma, terminal=True)
    else:
        g, grads, _ = V.chain_vjp(inv_layers, flags, y, None, lb, mu, scale_tril=L)
    assert rel(B.to_numpy(ybar), g) < 1e-3
    flow_grads = grads[::-1]  # flow order
    for k in (0, 3):
        for name in ("W", "c"):
            assert rel(fgrads[k][name].cpu().numpy(), flow_grads[k][name]) < 1e-3, (k, name)


def test_rand_and_host_path(B):
    import torch

    rng = np.random.default_rng(41)
    D, N = 16, 3001
    flow, ora = _flow(B, rng, D)
    td = B.transformed(B.MvNormal(D), flow)
    y, lj = B.rand(td, N, seed=77, offset=2, with_logjac=True)
    z = O.philox_normals(77, 2, D, N)
    y64, l64 = O.chain_forward(ora, z.astype(np.float64))
    y32, l32 = O.chain_forward(ora, z.astype(f32))
    gate(B.to_numpy(y), y64, y32, "rand y")
    gate(B.to_numpy(lj), l64, l32, "rand logjac")
    x = B.rand(td.dist, N, seed=77, offset=2)
    y2, lj2 = B.run_chain(flow, x)
    assert B.to_numpy(y).tobytes() == B.to_numpy(y2).tobytes() and B.to_numpy(lj).tobytes() == B.to_numpy(lj2).tobytes()
    # host-buffer path: bit-identical to the device path
    xh = B.from_numpy(B.to_numpy(x), device="cpu")
    yh, ljh = B.run_chain(flow, xh)
    assert np.asarray(yh).tobytes() == B.to_numpy(y2).tobytes() or B.to_numpy(yh).tobytes() == B.to_numpy(y2).tobytes()
    assert B.to_numpy(ljh).tobytes() == B.to_numpy(lj2).tobytes()
    lp_dev = B.to_numpy(B.logpdf(td, y2))
    lp_host = B.to_numpy(B.logpdf(td, B.from_numpy(B.to_numpy(y2), device="cpu")))
    assert lp_dev.tobytes() == lp_host.tobytes()
    del torch


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,n1,n2,K,N,with_c", [(2, 1, 1, 2, 300, True), (10, 4, 3, 5, 777, False), (40, 20, 20, 8, 1500, True),
                                                 (136, 128, 8, 16, 200, True), (256, 128, 128, 4, 150, True)])
def test_vjp(B, D, n1, n2, K, N, with_c, inv):
    import torch

    rng = np.random.default_rng(D + 3 * K + N + inv)
    Bv = 2.5
    idx1, idx2, Wm, c = spec(rng, D, n1, n2, K, scattered=True, with_c=with_c)
    x = batch(rng, D, N, Bv)
    yb = rng.standard_normal((D, N)).astype(f32)
    lb = rng.standard_normal(N).astype(f32)
    lay = layer(B, D, idx1, idx2, Wm, c, K, Bv)
    t = B.inverse(lay) if inv else lay
    xbar, grads = B.chain_vjp(t, B.from_numpy(x), B.from_numpy(yb), torch.from_numpy(lb).cuda())
    xb64, W64, c64 = S.vjp(idx1, idx2, Wm, c, K, Bv, x, yb, lb, inverse=inv)
    xb32, W32, c32 = S.vjp(idx1, idx2, Wm, c, K, Bv, x, yb, lb, inverse=inv, dtype=f32)
    gate(B.to_numpy(xbar), xb64, xb32, "xbar")
    gate(grads[0]["W"].cpu().numpy(), W64, W32, "Wbar")
    if with_c:
        gate(grads[0]["c"].cpu().numpy(), c64, c32, "cbar")
    else:
        assert "c" not in grads[0]


def test_vjp_repeatable_graph_and_empty(B):
    import torch

    rng = np.random.default_rng(61)
    D, N, K = 24, 5000, 8
    flow, _ = _flow(B, rng, D, K)
    x = B.from_numpy(batch(rng, D, N, 2.0))
    yb = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lb = torch.randn(N, device="cuda")
    a = B.chain_vjp(flow, x, yb, lb)
    b = B.chain_vjp(flow, x, yb, lb)
    assert torch.equal(a[0], b[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], b[1]) for k in p)
    out = {}
    g = B.GraphedCalls(lambda: out.__setitem__("r", B.chain_vjp(flow, x, yb, lb)))
    cr = out["r"]
    cr[0].fill_(float("nan"))
    g()
    torch.cuda.synchronize()
    assert torch.equal(a[0], cr[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], cr[1]) for k in p)
    # N = 0 zeroes the requested cotangents
    e = B.colmajor_empty(D, 0, "cuda")
    _, ge = B.chain_vjp(flow, e)
    assert all(float(t.abs().sum()) == 0 for gg in ge for t in gg.values())


def _desc(B, D, n1, n2, K, Bv=2.0, with_c=True, inverse=0):
    import torch

    J = 3 * K - 1
    W = torch.zeros((max(J * n1 * n2, 1),), device="cuda")
    c = torch.zeros((max(J * n1, 1),), device="cuda")
    i1 = torch.arange(n1, dtype=torch.int32, device="cuda")
    i2 = torch.arange(n1, n1 + n2, dtype=torch.int32, device="cuda") % max(D, 1)
    d = B._lib.LayerDesc()
    d.kind, d.inverse = B._lib.COUPLING_RQS, inverse
    d.n0, d.n1, d.n2, d.n3, d.f0 = n1, n2, K, 0, Bv
    d.p0, d.p1, d.i0, d.i1 = W.data_ptr(), c.data_ptr() if with_c else None, i1.data_ptr(), i2.data_ptr()
    return d, (W, c, i1, i2)


def test_slot_status_codes(B):
    import torch

    L = B.lib()
    D, N = 8, 64
    x = torch.zeros((N * D,), device="cuda")
    xb = torch.zeros((N * D,), device="cuda")
    for with_c, slot, want in [(True, 2, -2), (True, 3, -2), (False, 1, -1), (True, 1, 0), (True, 0, 0)]:
        d, keep = _desc(B, D, 4, 4, 3, with_c=with_c)
        arr = (B._lib.LayerDesc * 1)(d)
        bar = torch.zeros((4 * 3 * 8 * 4,), device="cuda")
        ptrs = (ctypes.c_void_p * 4)()
        ptrs[slot] = bar.data_ptr()
        wsb = L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
        ws = torch.empty((wsb,), dtype=torch.uint8, device="cuda")
        rc = L.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D,
                                 D, ws.data_ptr(), wsb, stream())
        assert rc == want, (with_c, slot, rc)
    torch.cuda.synchronize()


@pytest.mark.parametrize("D,n1,n2,K", [(300, 129, 1, 2), (300, 1, 129, 2), (40, 4, 4, 17), (1025, 4, 4, 2), (40, 4, 4, 1)])
def test_past_the_envelope(B, D, n1, n2, K):
    import torch

    L = B.lib()
    N = 100
    d, keep = _desc(B, D, n1, n2, K)
    arr = (B._lib.LayerDesc * 1)(d)
    x = torch.zeros((N * D,), device="cuda")
    y = torch.full((N * D,), 3.5, device="cuda")
    lj = torch.full((N,), 3.5, device="cuda")
    xb = torch.full((N * D,), 3.5, device="cuda")
    torch.cuda.synchronize()
    assert L.b2b_chain_workspace_bytes(arr, 1, D, N, 1, 0) == 0
    assert L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N) == 0
    assert L.b2b_chain_run_f32(arr, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream()) == -2
    assert L.b2b_last_launch_count() == 0
    assert L.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, None, 0, stream()) == -2
    assert L.b2b_last_launch_count() == 0
    torch.cuda.synchronize()
    assert (y == 3.5).all() and (lj == 3.5).all() and (xb == 3.5).all()


def test_envelope_corners_run(B):
    """The largest shapes inside the envelope run (n1 = n2 = 128, K = 16, D = 1024), forward and reverse."""
    import torch

    rng = np.random.default_rng(71)
    D, N, K = 1024, 300, 16
    idx1, idx2, Wm, c = spec(rng, D, 128, 128, K, scattered=True)
    x = batch(rng, D, N, 3.0)
    lay = layer(B, D, idx1, idx2, Wm, c, K, 3.0)
    y, lj = B.with_logabsdet_jacobian(lay, B.from_numpy(x))
    cols = [0, 7, N - 1]
    y64, l64 = S.forward(idx1, idx2, Wm, c, K, 3.0, x.astype(np.float64), np.float64, cols)
    y32, l32 = S.forward(idx1, idx2, Wm, c, K, 3.0, x, f32, cols)
    gate(B.to_numpy(y)[:, cols], y64, y32, "y")
    gate(B.to_numpy(lj)[cols], l64, l32, "lj")
    xbar, g = B.chain_vjp(lay, B.from_numpy(x), None, torch.ones(N, device="cuda"))
    xb64, W64, c64 = S.vjp(idx1, idx2, Wm, c, K, 3.0, x, None, np.ones(N))
    xb32, W32, c32 = S.vjp(idx1, idx2, Wm, c, K, 3.0, x, None, np.ones(N), dtype=f32)
    gate(B.to_numpy(xbar), xb64, xb32, "xbar")
    gate(g[0]["W"].cpu().numpy(), W64, W32, "Wbar")
    gate(g[0]["c"].cpu().numpy(), c64, c32, "cbar")


def test_float64_descriptor_unsupported(B):
    import torch

    L = B.lib()
    D, N = 8, 16
    d = B._lib.LayerDesc64()
    W = torch.zeros(8 * 4 * 4, dtype=torch.float64, device="cuda")
    i = torch.arange(8, dtype=torch.int32, device="cuda")
    d.kind, d.n0, d.n1, d.n2, d.f0 = B._lib.COUPLING_RQS, 4, 4, 3, 2.0
    d.p0, d.i0, d.i1 = W.data_ptr(), i.data_ptr(), i[4:].data_ptr()
    arr = (B._lib.LayerDesc64 * 1)(d)
    x = torch.zeros(D * N, dtype=torch.float64, device="cuda")
    y = torch.zeros(D * N, dtype=torch.float64, device="cuda")
    assert L.b2b_chain_run_f64(arr, 1, x.data_ptr(), y.data_ptr(), None, None, D, N, D, D, 0, None, 0, stream()) == -2
    assert L.b2b_chain_vjp_workspace_bytes_f64(arr, 1, D, N) == 0
    assert L.b2b_chain_vjp_f64(arr, 1, x.data_ptr(), None, None, y.data_ptr(), None, D, N, D, D, D, None, 0, stream()) == -2


def test_training_lowers_nll_and_first_gradient(B):
    """A 4-block spline flow at D = 8 trained with Adam on seeded data: the first-step gradient matches the oracle and
    the NLL goes down."""
    import torch

    rng = np.random.default_rng(81)
    D, N, K, Bv = 8, 4096, 6, 4.0
    blocks, ora = [], []
    for k in range(4):
        rows = np.roll(np.arange(1, D + 1), k)
        i1, i2 = [int(r) for r in rows[: D // 2]], [int(r) for r in rows[D // 2:]]
        Wm = (rng.standard_normal(((3 * K - 1) * len(i1), len(i2))) * 0.1).astype(f32)
        c = (rng.standard_normal((3 * K - 1) * len(i1)) * 0.1).astype(f32)
        blocks.append(layer(B, D, i1, i2, Wm, c, K, Bv))
        ora.append(S.SplineLayer(i1, i2, Wm, c, K, Bv))
    flow = B.autograd.Flow(B.Composed(*blocks))
    z = rng.standard_normal((D, N))
    data = np.stack([z[0] * 1.5, z[1] * 0.5 + 0.3 * z[0] ** 2] + [z[j] * (0.5 + 0.1 * j) for j in range(2, D)]).astype(f32)
    y = B.from_numpy(data)
    nll = flow.nll(y)
    nll.backward()
    # oracle: −Σ logpdf through inverse(flow) and the standard-normal base
    inv_layers, inputs, cur = ora[::-1], [], data.astype(np.float64)
    lj = 0.0
    for lay in inv_layers:
        inputs.append(cur)
        cur, l = lay.inverse(cur)
        lj = lj + l
    lp = O.mvnormal_diag_logpdf(None, None, cur) + lj
    assert abs(float(nll) + lp.sum()) <= 1e-4 * abs(lp.sum())
    g = V.mvnormal_diag_logpdf_vjp(np.zeros(D), np.ones(D), cur, -np.ones(N))[0]
    grads = [None] * 4
    for l in reversed(range(4)):
        g, grads[l] = inv_layers[l].vjp(inputs[l], g, -np.ones(N), inverse=True)
    grads = grads[::-1]
    for k in range(4):
        Wp, cp = flow.params[2 * k], flow.params[2 * k + 1]
        assert rel(Wp.grad.cpu().numpy().T, grads[k]["W"]) < 1e-3
        assert rel(cp.grad.cpu().numpy(), grads[k]["c"]) < 1e-3
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    first = float(nll)
    for _ in range(40):
        opt.zero_grad()
        loss = flow.nll(y)
        loss.backward()
        opt.step()
    assert float(flow.nll(y)) < first - 0.02 * abs(first)
