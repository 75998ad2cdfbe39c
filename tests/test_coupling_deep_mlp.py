"""GPU tests of the deep neural-network coupling layer, B2B_COUPLING_DEEP_MLP: Coupling(x₂ -> Shift(t) ∘ Scale(exp.(s)),
mask) with [s; t] from an MLP of M = 2..4 hidden layers, against the float64 reference of
tests/coupling_deep_mlp_oracle.py.  Gates are tied to the reference's own float32 error on the same input, as in
test_gpu_parity.gate: max(1e-5, k × ‖oracle32 − oracle64‖ / ‖oracle64‖), norm-wise, k = 2 for the forward pass.  Reverse
mode uses k = 4: the device sums each GEMM of the stack in a fixed sequential order and numpy in blocks, and the stack
puts up to five such GEMMs in series."""
import ctypes

import numpy as np
import pytest

import chain_vjp_oracle as V
import coupling_deep_mlp_oracle as DM
import coupling_mlp_oracle as M
import mvnormal_tril_oracle as T
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5
ACTS = [("tanh", 0.0), ("leaky_relu", 0.1)]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(dev, a64, a32, what="", k=2.0):
    tol = max(RTOL, k * rel(a32, a64))
    e = rel(dev, a64)
    assert e <= tol, (what, e, tol)


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def spec(rng, D, n1, n2, H, M, scattered=False, with_c=True, scale=0.8):
    """(idx1, idx2, weights, biases) with weights scaled so that every layer's pre-activation is O(1)."""
    rows = (rng.permutation(D) if scattered else np.arange(D)) + 1
    idx1, idx2 = [int(i) for i in rows[:n1]], [int(i) for i in rows[n1:n1 + n2]]
    weights = [(rng.standard_normal((H, n2)) * scale / np.sqrt(n2)).astype(f32)]
    weights += [(rng.standard_normal((H, H)) * 1.2 / np.sqrt(H)).astype(f32) for _ in range(M - 1)]
    weights += [(rng.standard_normal((2 * n1, H)) * scale / np.sqrt(H)).astype(f32)]
    biases = None
    if with_c:
        biases = [(rng.standard_normal(H) * 0.3).astype(f32) for _ in range(M)] + [(rng.standard_normal(2 * n1) * 0.2).astype(f32)]
    return idx1, idx2, weights, biases


def layer(B, D, idx1, idx2, weights, biases, act="tanh", slope=0.0):
    return B.Coupling(B.DeepMLPConditioner(weights, biases, activation=act, slope=slope), B.PartitionMask(D, idx1, idx2))


def stream():
    from bijectors_jl_b200.interface import _stream

    return _stream()


# D, n1, n2, H, scattered (x₃ rows exist whenever n1 + n2 < D)
SHAPES = [(3, 1, 1, 1, False), (10, 3, 5, 7, True), (64, 32, 32, 64, False), (200, 60, 100, 33, True),
          (1024, 128, 128, 128, True)]


def _parity(B, D, n1, n2, H, M, scattered, N, act, slope, inv, with_c):
    rng = np.random.default_rng(D * 7 + n1 + H + N + inv + 13 * M)
    sp = spec(rng, D, n1, n2, H, M, scattered, with_c=with_c)
    x = rng.standard_normal((D, N)).astype(f32)
    lay = layer(B, D, *sp, act, slope)
    y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, B.from_numpy(x))
    y, lj = B.to_numpy(y), B.to_numpy(lj)
    f = DM.inverse if inv else DM.forward
    sel = slice(None) if N <= 4097 else np.unique(np.r_[0, 1, N - 1, rng.integers(0, N, 300)])
    y64, l64 = f(*sp, act, slope, x[:, sel].astype(np.float64))
    y32, l32 = f(*sp, act, slope, x[:, sel], f32)
    r1 = np.asarray(sp[0]) - 1
    gate(y[r1][:, sel], y64[r1], y32[r1], "y1")
    gate(lj[sel], l64, l32, "logjac")
    rest = np.setdiff1d(np.arange(D), r1)
    assert y[rest].tobytes() == x[rest].tobytes()  # x₂ and x₃ bit-exact, whole batch
    assert np.isfinite(y).all() and np.isfinite(lj).all()


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
@pytest.mark.parametrize("M", [2, 3, 4])
@pytest.mark.parametrize("D,n1,n2,H,scattered", SHAPES)
def test_parity(B, D, n1, n2, H, scattered, M, act, slope, inv):
    for N in (1, 33, 4097):
        _parity(B, D, n1, n2, H, M, scattered, N, act, slope, inv, with_c=(N != 33))  # N = 33: no biases


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("M", [2, 4])
@pytest.mark.parametrize("D,n1,n2,H,scattered", [(64, 32, 32, 64, False), (1024, 128, 128, 128, True)])
def test_parity_large_batch(B, D, n1, n2, H, scattered, M, inv):
    _parity(B, D, n1, n2, H, M, scattered, (1 << 20) + 3, "tanh", 0.0, inv, with_c=True)


@pytest.mark.parametrize("act,slope", ACTS + [("leaky_relu", 0.0)])
def test_inverse_of_forward(B, act, slope):
    rng = np.random.default_rng(3)
    D, N = 48, 2000
    sp = spec(rng, D, 20, 24, 40, 3, scattered=True)
    x = rng.standard_normal((D, N)).astype(f32)
    lay = layer(B, D, *sp, act, slope)
    y, lj = B.with_logabsdet_jacobian(lay, B.from_numpy(x))
    xr, ljr = B.with_logabsdet_jacobian(B.inverse(lay), y)
    assert rel(B.to_numpy(xr), x) < 1e-6
    assert B.to_numpy(ljr).tobytes() == (-B.to_numpy(lj)).tobytes()  # the same Σ s, negated


def _raw(B, lay, inv, D, N, x, ldx, xoff, y, ldy, yoff, lj, acc):
    import torch

    from bijectors_jl_b200.interface import _desc_array

    arr = _desc_array(lay._descs(inv, D))
    L = B.lib()
    p = lambda t, off=0: None if t is None else t.data_ptr() + 4 * off  # noqa: E731
    rc = L.b2b_chain_run_f32(arr, 1, p(x, xoff), p(y, yoff), p(lj), None, D, N, ldx, ldy, acc, None, 0, stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("inv", [False, True])
def test_layouts(B, inv):
    """Padded ld, misaligned bases, in place, accumulate and logjac only give the bits of the plain call."""
    import torch

    rng = np.random.default_rng(11 + inv)
    D, N = 10, 333
    sp = spec(rng, D, 4, 3, 8, 3, scattered=True)
    x = rng.standard_normal((D, N)).astype(f32)
    lay = layer(B, D, *sp)
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
    base = torch.randn(N, device="cuda")
    lj.copy_(base)
    assert _raw(B, lay, inv, D, N, xb, ld, 1, yb, ld, 3, lj, 1) == 0  # accumulate
    assert lj.cpu().numpy().tobytes() == (base.cpu().numpy() + l0).astype(f32).tobytes()
    lj.fill_(0)
    assert _raw(B, lay, inv, D, N, xb, ld, 1, None, D, 0, lj, 0) == 0  # logjac only
    assert lj.cpu().numpy().tobytes() == l0.tobytes()
    assert _raw(B, lay, inv, D, N, xb, ld, 1, xb, ld, 1, lj, 0) == 0  # in place
    assert xv[:, :D].cpu().numpy().T.tobytes() == y0.tobytes()
    assert (xv[:, D:] == sentinel).all() and lj.cpu().numpy().tobytes() == l0.tobytes()


@pytest.mark.parametrize("inv", [False, True])
def test_slope_one_equals_the_affine_coupling(B, inv):
    """LeakyReLU(1) is the identity: the layer equals COUPLING_AFFINE on the folded product of its matrices."""
    rng = np.random.default_rng(5 + inv)
    D, N = 40, 3000
    idx1, idx2, weights, biases = spec(rng, D, 16, 20, 24, 3, scattered=True)
    x = rng.standard_normal((D, N)).astype(f32)
    deep = layer(B, D, idx1, idx2, weights, biases, "leaky_relu", 1.0)
    Wc, cc = weights[0].astype(np.float64), biases[0].astype(np.float64)
    for W, c in zip(weights[1:], biases[1:]):
        Wc, cc = W.astype(np.float64) @ Wc, W.astype(np.float64) @ cc + c
    aff = B.Coupling(B.AffineConditioner(Wc.astype(f32), cc.astype(f32)), B.PartitionMask(D, idx1, idx2))
    run = lambda l: [B.to_numpy(a) for a in B.with_logabsdet_jacobian(B.inverse(l) if inv else l, B.from_numpy(x))]  # noqa: E731
    (ym, lm), (ya, la) = run(deep), run(aff)
    f = O.coupling_affine_inverse if inv else O.coupling_affine_forward
    y64, l64 = f(idx1, idx2, Wc, cc, x.astype(np.float64))
    y32, l32 = (DM.inverse if inv else DM.forward)(idx1, idx2, weights, biases, "leaky_relu", 1.0, x, f32)
    gate(ym, y64, y32, "y")
    gate(lm, l64, l32, "logjac")
    assert rel(ym, ya) < 3e-5 and rel(lm, la) < 3e-5  # both within the gate of the float64 result


@pytest.mark.parametrize("inv", [False, True])
def test_exact_reduction_to_the_one_hidden_layer_kind(B, inv):
    """M = 2 with W_2 = I, c_2 = 0 and ReLU (LeakyReLU slope 0): h_2 = relu(h_1) = h_1, so the layer is
    B2B_COUPLING_MLP on the same W_in, c_1, W_out, c_out -- bit for bit, since layer 1 and the affine law are that
    kind's own code and each h_2 is an fmaf chain of exact products."""
    rng = np.random.default_rng(17 + inv)
    D, N, H = 40, 3001, 24
    idx1, idx2, weights, biases = spec(rng, D, 16, 20, H, 2, scattered=True)
    weights[1] = np.eye(H, dtype=f32)
    biases[1] = np.zeros(H, f32)
    assert np.abs(biases[2]).min() > 0  # c_out nonzero: no sum of the output layer starts at a signed zero
    x = rng.standard_normal((D, N)).astype(f32)
    deep = layer(B, D, idx1, idx2, weights, biases, "leaky_relu", 0.0)
    mlp = B.Coupling(B.MLPConditioner(weights[0], biases[0], weights[2], biases[2], activation="leaky_relu", slope=0.0),
                     B.PartitionMask(D, idx1, idx2))
    run = lambda l: [B.to_numpy(a) for a in B.with_logabsdet_jacobian(B.inverse(l) if inv else l, B.from_numpy(x))]  # noqa: E731
    (yd, ld), (ym, lm) = run(deep), run(mlp)
    assert yd.tobytes() == ym.tobytes() and ld.tobytes() == lm.tobytes()


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
@pytest.mark.parametrize("M", [2, 3, 4])
@pytest.mark.parametrize("D,n1,n2,H,N,with_c,cots", [
    (3, 1, 1, 1, 300, True, "yl"), (10, 3, 5, 7, 777, False, "yl"), (40, 20, 20, 33, 1500, True, "y"),
    (64, 32, 32, 64, 5000, True, "l"), (200, 60, 100, 33, 200, True, "yl"), (1024, 128, 128, 128, 150, True, "yl")])
def test_vjp(B, D, n1, n2, H, N, with_c, cots, M, act, slope, inv):
    import torch

    rng = np.random.default_rng(D + 3 * H + N + inv + 17 * M)
    sp = spec(rng, D, n1, n2, H, M, scattered=True, with_c=with_c)
    x = rng.standard_normal((D, N)).astype(f32)
    yb = rng.standard_normal((D, N)).astype(f32) if "y" in cots else None
    lb = rng.standard_normal(N).astype(f32) if "l" in cots else None
    lay = layer(B, D, *sp, act, slope)
    t = B.inverse(lay) if inv else lay
    xbar, grads = B.chain_vjp(t, B.from_numpy(x), None if yb is None else B.from_numpy(yb),
                              None if lb is None else torch.from_numpy(lb).cuda())
    xb64, g64 = DM.vjp(*sp, act, slope, x, yb, lb, inverse=inv)
    xb32, g32 = DM.vjp(*sp, act, slope, x, yb, lb, inverse=inv, dtype=f32)
    gate(B.to_numpy(xbar), xb64, xb32, "xbar", k=4.0)
    names = ("W_in", "W_hid", "W_out", "c") if with_c else ("W_in", "W_hid", "W_out")
    assert set(grads[0]) == set(names)
    assert tuple(grads[0]["W_hid"].shape) == (M - 1, H, H)
    for k in names:
        gate(grads[0][k].cpu().numpy(), g64[k], g32[k], k + "bar", k=4.0)


def _flow(B, rng, D, H=12):
    """Deep coupling (tanh, M = 3) ∘ BatchNorm ∘ Permute ∘ one-hidden-layer coupling ∘ deep coupling (LeakyReLU,
    M = 2) ∘ Planar, device and oracle layers (application order)."""
    dev, ora = [], []
    sp = spec(rng, D, D // 2, D - D // 2, H, 3)
    dev.append(layer(B, D, *sp))
    ora.append(DM.DeepMLPLayer(*sp))
    b, logs = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
    m, v = (rng.standard_normal(D) * 0.1).astype(f32), (rng.uniform(0.5, 1.5, D)).astype(f32)
    dev.append(B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v))
    ora.append(O.Layer("batchnorm", dict(bn=O.BatchNormParams(b=b, logs=logs, m=m, v=v, eps=1e-5))))
    perm = rng.permutation(D) + 1
    dev.append(B.Permute(perm))
    ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))))
    rows = rng.permutation(D) + 1
    i1, i2 = [int(r) for r in rows[: D // 4]], [int(r) for r in rows[D // 4:]]
    W1 = (rng.standard_normal((H, len(i2))) * 0.8 / np.sqrt(len(i2))).astype(f32)
    W2 = (rng.standard_normal((2 * len(i1), H)) * 0.8 / np.sqrt(H)).astype(f32)
    c1, c2 = (rng.standard_normal(H) * 0.3).astype(f32), (rng.standard_normal(2 * len(i1)) * 0.2).astype(f32)
    dev.append(B.Coupling(B.MLPConditioner(W1, c1, W2, c2), B.PartitionMask(D, i1, i2)))
    ora.append(M.MLPLayer(i1, i2, W1, c1, W2, c2))
    sp = spec(rng, D, D // 3, D - D // 3 - 1, H + 1, 2, scattered=True)
    dev.append(layer(B, D, *sp, "leaky_relu", 0.2))
    ora.append(DM.DeepMLPLayer(*sp, "leaky_relu", 0.2))
    w, u = (rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32)
    bb = rng.standard_normal(1).astype(f32)
    dev.append(B.PlanarLayer(w, u, bb))
    ora.append(O.Layer("planar", dict(w=w, u=u, b=bb)))
    return B.Composed(*dev), ora


DEEP_IN_FLOW = (0, 4)  # positions of the deep couplings in _flow


def test_chain_forward_inverse(B):
    rng = np.random.default_rng(21)
    D, N = 16, 700
    flow, ora = _flow(B, rng, D)
    x = rng.standard_normal((D, N)).astype(f32)
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


def test_chain_vjp(B):
    """chain_vjp through the whole mixed flow: x̄ and every cotangent of both deep couplings and the kind-13 coupling."""
    import torch

    rng = np.random.default_rng(23)
    D, N = 16, 900
    flow, ora = _flow(B, rng, D)
    x = rng.standard_normal((D, N)).astype(f32)
    yb = rng.standard_normal((D, N)).astype(f32)
    lb = rng.standard_normal(N).astype(f32)
    xbar, grads = B.chain_vjp(flow, B.from_numpy(x), B.from_numpy(yb), torch.from_numpy(lb).cuda())
    flags = [False] * len(ora)
    g64, gr64, _ = V.chain_vjp(ora, flags, x, yb, lb)
    g32, gr32, _ = V.chain_vjp(ora, flags, x, yb, lb, dtype=f32)
    tol = lambda a32, a64: max(3e-4, 4 * rel(a32, a64))  # noqa: E731
    assert rel(B.to_numpy(xbar), g64) <= tol(g32, g64)
    for k in DEEP_IN_FLOW:
        assert set(grads[k]) == {"W_in", "W_hid", "W_out", "c"}
        for name in grads[k]:
            assert rel(grads[k][name].cpu().numpy(), gr64[k][name]) <= tol(gr32[k][name], gr64[k][name]), (k, name)
    for name in ("W1", "c1", "W2", "c2"):
        assert rel(grads[3][name].cpu().numpy(), gr64[3][name]) <= tol(gr32[3][name], gr64[3][name]), name


@pytest.mark.parametrize("base", ["diag", "tril"])
def test_logpdf_and_vjp(B, base):
    import torch

    rng = np.random.default_rng(31 + (base == "tril"))
    D, N = 16, 600
    flow, ora = _flow(B, rng, D)
    y = rng.standard_normal((D, N)).astype(f32)
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

    def chain_lp(yy, dt):
        cur, lj = np.asarray(yy, dt), 0.0
        for lay in inv_layers:
            cur, l = lay.inverse(cur)
            lj = lj + l
        if base == "diag":
            return O.mvnormal_diag_logpdf(mu.astype(dt), sigma.astype(dt), cur) + lj
        return T.logpdf(L, mu, cur, dt) + lj

    lp64, lp32 = chain_lp(y, np.float64), chain_lp(y, f32)
    gate(lp, lp64, lp32, "logpdf")
    s, lps = B.logpdf_sum(td, yd)
    assert B.to_numpy(lps).tobytes() == lp.tobytes()
    assert abs(float(s) - lp64.sum()) <= max(1e-5, 2 * abs(lp32.sum(dtype=np.float64) - lp64.sum())) * abs(lp64.sum()) + 1e-3
    # reverse mode: ȳ and the cotangents of both deep couplings
    lb = rng.standard_normal(N)
    ybar, fgrads, _ = B.logpdf_vjp(td, yd, torch.from_numpy(lb.astype(f32)).cuda())
    flags = [True] * len(inv_layers)
    if base == "diag":
        g, grads, _ = V.chain_vjp(inv_layers, flags, y, None, lb, mu, sigma, terminal=True)
    else:
        g, grads, _ = V.chain_vjp(inv_layers, flags, y, None, lb, mu, scale_tril=L)
    assert rel(B.to_numpy(ybar), g) < 3e-4
    flow_grads = grads[::-1]  # flow order
    for k in DEEP_IN_FLOW:
        for name in ("W_in", "W_hid", "W_out", "c"):
            assert rel(fgrads[k][name].cpu().numpy(), flow_grads[k][name]) < 3e-4, (k, name)


def test_rand_and_host_path(B):
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
    assert B.to_numpy(yh).tobytes() == B.to_numpy(y2).tobytes()
    assert B.to_numpy(ljh).tobytes() == B.to_numpy(lj2).tobytes()
    lp_dev = B.to_numpy(B.logpdf(td, y2))
    lp_host = B.to_numpy(B.logpdf(td, B.from_numpy(B.to_numpy(y2), device="cpu")))
    assert lp_dev.tobytes() == lp_host.tobytes()


def test_repeatable_graph_and_empty(B):
    import torch

    rng = np.random.default_rng(61)
    D, N = 24, 5000
    flow, _ = _flow(B, rng, D)
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    yb = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lb = torch.randn(N, device="cuda")
    f0, f1 = B.run_chain(flow, x), B.run_chain(flow, x)
    assert torch.equal(f0[0], f1[0]) and torch.equal(f0[1], f1[1])
    a = B.chain_vjp(flow, x, yb, lb)
    b = B.chain_vjp(flow, x, yb, lb)
    assert torch.equal(a[0], b[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], b[1]) for k in p)
    out = {}
    g = B.GraphedCalls(lambda: out.update(f=B.run_chain(flow, x), r=B.chain_vjp(flow, x, yb, lb)))
    cf, cr = out["f"], out["r"]
    cf[0].fill_(float("nan"))
    cr[0].fill_(float("nan"))
    g()
    torch.cuda.synchronize()
    assert torch.equal(f0[0], cf[0]) and torch.equal(f0[1], cf[1])
    assert torch.equal(a[0], cr[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], cr[1]) for k in p)
    # N = 0 zeroes the requested cotangents
    e = B.colmajor_empty(D, 0, "cuda")
    _, ge = B.chain_vjp(flow, e)
    assert all(float(t.abs().sum()) == 0 for gg in ge for t in gg.values())


def _desc(B, D, n1, n2, H, M, act=0, with_c=True, inverse=0):
    import torch

    W_in = torch.zeros((max(H * n2, 1),), device="cuda")
    W_hid = torch.zeros((max((M - 1) * H * H, 1),), device="cuda")
    W_out = torch.zeros((max(2 * n1 * H, 1),), device="cuda")
    c = torch.zeros((max(M * H + 2 * n1, 1),), device="cuda")
    i1 = torch.arange(n1, dtype=torch.int32, device="cuda")
    i2 = torch.arange(n1, n1 + n2, dtype=torch.int32, device="cuda") % max(D, 1)
    d = B._lib.LayerDesc()
    d.kind, d.inverse = B._lib.COUPLING_DEEP_MLP, inverse
    d.n0, d.n1, d.n2, d.n3, d.f0 = n1, n2, H, act | (M << 8), 0.1
    d.p0, d.p1, d.p2, d.i0, d.i1 = W_in.data_ptr(), W_hid.data_ptr(), W_out.data_ptr(), i1.data_ptr(), i2.data_ptr()
    d.p3 = c.data_ptr() if with_c else None
    return d, (W_in, W_hid, W_out, c, i1, i2)


def test_slot_status_codes(B):
    """Every slot with c given; without c, W̄_in, W̄_hid and W̄_out work and a c̄ request is B2B_EINVAL with x̄ untouched."""
    import torch

    L = B.lib()
    D, N = 8, 64
    x = torch.zeros((N * D,), device="cuda")
    for with_c, slot, want in [(True, 0, 0), (True, 1, 0), (True, 2, 0), (True, 3, 0), (False, 3, -1),
                               (False, 0, 0), (False, 1, 0), (False, 2, 0)]:
        d, keep = _desc(B, D, 4, 4, 3, 3, with_c=with_c)
        arr = (B._lib.LayerDesc * 1)(d)
        bar = torch.full((64,), float("nan"), device="cuda")
        xb = torch.full((N * D,), float("nan"), device="cuda")
        ptrs = (ctypes.c_void_p * 4)()
        ptrs[slot] = bar.data_ptr()
        wsb = L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
        ws = torch.empty((wsb,), dtype=torch.uint8, device="cuda")
        rc = L.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D,
                                 D, ws.data_ptr(), wsb, stream())
        torch.cuda.synchronize()
        assert rc == want, (with_c, slot, rc)
        if want == 0:  # the requested slot is written, nothing past it: W̄_in 12, W̄_hid 18, W̄_out 24, c̄ 17 floats
            n = (12, 18, 24, 17)[slot]
            assert torch.isfinite(bar[:n]).all() and torch.isnan(bar[n:]).all() and torch.isfinite(xb).all()
        else:
            assert L.b2b_last_launch_count() == 0 and torch.isnan(xb).all() and torch.isnan(bar).all()


@pytest.mark.parametrize("D,n1,n2,H,M,act,want", [(300, 129, 1, 4, 2, 0, -2), (300, 1, 129, 4, 2, 0, -2),
                                                  (40, 4, 4, 129, 2, 0, -2), (40, 4, 4, 4, 5, 1, -2),
                                                  (1025, 4, 4, 4, 2, 1, -2), (40, 4, 4, 4, 1, 0, -1),
                                                  (40, 4, 4, 4, 2, 2, -1)])
def test_refused_with_nothing_launched(B, D, n1, n2, H, M, act, want):
    import torch

    L = B.lib()
    N = 100
    d, keep = _desc(B, D, n1, n2, H, M, act)
    arr = (B._lib.LayerDesc * 1)(d)
    x = torch.zeros((N * D,), device="cuda")
    y = torch.full((N * D,), float("nan"), device="cuda")
    lj = torch.full((N,), float("nan"), device="cuda")
    xb = torch.full((N * D,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    if want == -2:
        assert L.b2b_chain_workspace_bytes(arr, 1, D, N, 1, 0) == 0
    assert L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N) == 0
    assert L.b2b_chain_run_f32(arr, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream()) == want
    assert L.b2b_last_launch_count() == 0
    assert L.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, None, 0, stream()) == want
    assert L.b2b_last_launch_count() == 0
    torch.cuda.synchronize()
    assert torch.isnan(y).all() and torch.isnan(lj).all() and torch.isnan(xb).all()


def test_float64_descriptor_unsupported(B):
    import torch

    L = B.lib()
    D, N = 8, 16
    d = B._lib.LayerDesc64()
    W = torch.zeros(8 * 4 * 4, dtype=torch.float64, device="cuda")
    i = torch.arange(8, dtype=torch.int32, device="cuda")
    d.kind, d.n0, d.n1, d.n2, d.n3 = B._lib.COUPLING_DEEP_MLP, 4, 4, 3, 2 << 8
    d.p0, d.p1, d.p2, d.i0, d.i1 = W.data_ptr(), W.data_ptr(), W.data_ptr(), i.data_ptr(), i[4:].data_ptr()
    arr = (B._lib.LayerDesc64 * 1)(d)
    x = torch.zeros(D * N, dtype=torch.float64, device="cuda")
    y = torch.zeros(D * N, dtype=torch.float64, device="cuda")
    assert L.b2b_chain_run_f64(arr, 1, x.data_ptr(), y.data_ptr(), None, None, D, N, D, D, 0, None, 0, stream()) == -2
    assert L.b2b_chain_vjp_workspace_bytes_f64(arr, 1, D, N) == 0
    assert L.b2b_chain_vjp_f64(arr, 1, x.data_ptr(), None, None, y.data_ptr(), None, D, N, D, D, D, None, 0, stream()) == -2
    with pytest.raises(TypeError):
        B.DeepMLPConditioner([np.zeros((3, 4)), np.zeros((3, 3)), np.zeros((8, 3))], dtype=torch.float64)


def test_training_lowers_nll_and_first_gradient(B):
    """A 4-block deep-MLP RealNVP at D = 8 (M = 2 and 3, both activations) trained with Adam on seeded data: the
    first-step gradient matches the oracle and the NLL goes down."""
    import torch

    rng = np.random.default_rng(81)
    D, N, H = 8, 4096, 16
    blocks, ora = [], []
    for k in range(4):
        rows = np.roll(np.arange(1, D + 1), 2 * k)
        i1, i2 = [int(r) for r in rows[: D // 2]], [int(r) for r in rows[D // 2:]]
        Mk = 2 + k % 2
        weights = [(rng.standard_normal((H, len(i2))) * 0.3).astype(f32)]
        weights += [(rng.standard_normal((H, H)) * 0.8 / np.sqrt(H)).astype(f32) for _ in range(Mk - 1)]
        weights += [(rng.standard_normal((2 * len(i1), H)) * 0.05).astype(f32)]
        biases = [(rng.standard_normal(H) * 0.1).astype(f32) for _ in range(Mk)] + [np.zeros(2 * len(i1), f32)]
        act = ("tanh", 0.0) if k < 2 else ("leaky_relu", 0.1)
        blocks.append(layer(B, D, i1, i2, weights, biases, *act))
        ora.append(DM.DeepMLPLayer(i1, i2, weights, biases, *act))
    flow = B.autograd.Flow(B.Composed(*blocks))
    assert len(flow.params) == 16
    z = rng.standard_normal((D, N))
    data = np.stack([z[0] * 1.5, z[1] * 0.5 + 0.3 * z[0] ** 2] + [z[j] * (0.5 + 0.1 * j) for j in range(2, D)]).astype(f32)
    y = B.from_numpy(data)
    nll = flow.nll(y)
    nll.backward()
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
        for i, name in enumerate(("W_in", "W_hid", "W_out", "c")):
            got = flow.params[4 * k + i].grad.cpu().numpy()
            got = np.swapaxes(got, -1, -2) if got.ndim >= 2 else got  # storage is column-major
            assert rel(got, grads[k][name]) < 3e-4, (k, name)
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    first = float(nll)
    for _ in range(40):
        opt.zero_grad()
        loss = flow.nll(y)
        loss.backward()
        opt.step()
    assert float(flow.nll(y)) < first - 0.02 * abs(first)
