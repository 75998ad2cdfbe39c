"""GPU tests of the deep neural spline coupling layer, B2B_COUPLING_DEEP_MLP_RQS: Coupling(x₂ -> RationalQuadraticSpline(…,
B), mask) whose raw knots come from an MLP with M = 2..4 hidden layers, against the float64 reference of
tests/coupling_deep_mlp_rqs_oracle.py.  Gates are tied to the reference's own float32 error on the same input, as in
test_coupling_mlp_rqs.py: 2× for the forward, 4× for reverse mode (the cotangents pass through M + 1 GEMMs, each summed
in a fixed fmaf order on the device and blocked by numpy), and max(3e-4, 4×) in chains, where the device recomputes
each layer's input in float32.  Reverse mode with LeakyReLU takes 16×: every hidden pre-activation that the device and
numpy round to opposite sides of 0 changes σ′ by 1 − slope, and M layers have M times as many of them as kind 14's one
(W̄_in came out 12× the float32 reference's error at M = 2, with tanh the same cases stay within 4×)."""
import ctypes

import numpy as np
import pytest

import chain_vjp_oracle as V
import coupling_deep_mlp_oracle as DM
import coupling_deep_mlp_rqs_oracle as DR
import coupling_mlp_rqs_oracle as R
import mvnormal_tril_oracle as T
import spline_coupling_oracle as S
import test_mixed_chains as MC
import test_vjp_training_batches as TB
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5
ACTS = [("tanh", 0.0), ("leaky_relu", 0.1)]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(dev, a64, a32, what="", k=2.0, floor=RTOL):
    tol = max(floor, k * rel(a32, a64))
    e = rel(dev, a64)
    assert e <= tol, (what, e, tol)


def vjp_gate(dev, a64, a32, what="", act="tanh"):
    gate(dev, a64, a32, what, k=4.0 if act == "tanh" else 16.0)


def chain_gate(dev, a64, a32, what=""):
    gate(dev, a64, a32, what, k=4.0, floor=3e-4)


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def spec(rng, D, n1, n2, H, M, K, Bv=3.0, scattered=False, with_c=True, scale=0.8):
    """(idx1, idx2, weights, biases, K, B): the oracle's positional arguments before the activation."""
    rows = (rng.permutation(D) if scattered else np.arange(D)) + 1
    idx1, idx2 = [int(i) for i in rows[:n1]], [int(i) for i in rows[n1:n1 + n2]]
    J = (3 * K - 1) * n1
    weights = [(rng.standard_normal((H, n2)) * scale / np.sqrt(n2)).astype(f32)]
    weights += [(rng.standard_normal((H, H)) * 1.2 / np.sqrt(H)).astype(f32) for _ in range(M - 1)]
    weights += [(rng.standard_normal((J, H)) * scale / np.sqrt(H)).astype(f32)]
    biases = None
    if with_c:
        biases = [(rng.standard_normal(H) * 0.3).astype(f32) for _ in range(M)] + [(rng.standard_normal(J) * 0.3).astype(f32)]
    return idx1, idx2, weights, biases, K, Bv


def batch(rng, D, N, Bv=3.0):
    """Uniform on [−B/0.95, B/0.95]: about 5 % of the elements lie outside the box.  Elements within 1e-6 of ±B are
    moved to 0 (the spline element's known NaN between −(last knot) and −B, DESIGN.md §8 item 10)."""
    x = rng.uniform(-Bv / 0.95, Bv / 0.95, (D, N)).astype(f32)
    x[np.abs(np.abs(x) - Bv) <= 1e-6] = 0.0
    return x


def layer(B, D, idx1, idx2, weights, biases, K, Bv, act="tanh", slope=0.0):
    cond = B.DeepMLPSplineConditioner(weights, biases, K=K, B=Bv, activation=act, slope=slope)
    return B.Coupling(cond, B.PartitionMask(D, idx1, idx2))


def stream():
    from bijectors_jl_b200.interface import _stream

    return _stream()


def ptr(t, off=0):
    return None if t is None else t.data_ptr() + 4 * off


def _parity(B, D, n1, n2, H, M, K, scattered, N, act, slope, inv, with_c, seed):
    rng = np.random.default_rng(seed)
    sp = spec(rng, D, n1, n2, H, M, K, scattered=scattered, with_c=with_c)
    x = batch(rng, D, N)
    lay = layer(B, D, *sp, act, slope)
    y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, B.from_numpy(x))
    y, lj = B.to_numpy(y), B.to_numpy(lj)
    f = DR.inverse if inv else DR.forward
    cols = sorted({0, N - 1} | {int(c) for c in rng.integers(0, N, min(N, 150))})
    y64, l64 = f(*sp, act, slope, x.astype(np.float64), cols=cols)
    y32, l32 = f(*sp, act, slope, x, f32, cols=cols)
    r1 = np.asarray(sp[0]) - 1
    gate(y[r1][:, cols], y64[r1], y32[r1], "y1")
    gate(lj[cols], l64, l32, "logjac")
    rest = np.setdiff1d(np.arange(D), r1)
    assert y[rest].tobytes() == x[rest].tobytes()  # x₂ and x₃ bit-exact, whole batch
    assert np.isfinite(y).all() and np.isfinite(lj).all()


# D, n1, n2, H, K, scattered (x₃ rows exist whenever n1 + n2 < D)
SHAPES = [(6, 2, 3, 1, 2, True), (64, 32, 32, 17, 8, False), (64, 20, 30, 64, 8, True), (256, 100, 120, 128, 16, False),
          (200, 60, 100, 40, 2, True)]


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
@pytest.mark.parametrize("M", [2, 3, 4])
@pytest.mark.parametrize("D,n1,n2,H,K,scattered", SHAPES)
def test_parity(B, D, n1, n2, H, K, scattered, M, act, slope, inv):
    _parity(B, D, n1, n2, H, M, K, scattered, 1000, act, slope, inv, with_c=(H != 17),
            seed=D * 7 + n1 + H + K + M + inv + len(act))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("M", [2, 4])
@pytest.mark.parametrize("D,n1,n2,H,K,scattered,N", [(1024, 128, 128, 128, 16, True, 4099),
                                                     (64, 32, 32, 64, 8, False, 65539)])
def test_parity_envelope_corner_and_large_batch(B, D, n1, n2, H, K, scattered, N, M, inv):
    _parity(B, D, n1, n2, H, M, K, scattered, N, "tanh", 0.0, inv, with_c=True, seed=D + M + inv)


@pytest.mark.parametrize("act,slope", ACTS + [("leaky_relu", 0.0)])
def test_inverse_of_forward(B, act, slope):
    rng = np.random.default_rng(3)
    D, N = 48, 2000
    sp = spec(rng, D, 20, 24, 40, 3, 8, scattered=True)
    x = batch(rng, D, N)
    lay = layer(B, D, *sp, act, slope)
    y, lj = B.with_logabsdet_jacobian(lay, B.from_numpy(x))
    xr, ljr = B.with_logabsdet_jacobian(B.inverse(lay), y)
    assert rel(B.to_numpy(xr), x) < 1e-5
    assert rel(B.to_numpy(ljr), -B.to_numpy(lj)) < 1e-4


@pytest.mark.parametrize("inv", [False, True])
def test_exact_reduction_to_the_one_hidden_layer_kind(B, inv):
    """M = 2 with W_2 = I, c_2 = 0 and ReLU (LeakyReLU slope 0): h_2 = relu(h_1) = h_1, so the layer is
    B2B_COUPLING_MLP_RQS on the same W_in, c_1, W_out, c_out -- bit for bit, since layer 1 and the row loop are that
    kind's own code and each h_2 is an fmaf chain of exact products."""
    rng = np.random.default_rng(17 + inv)
    D, N, H, K = 40, 3001, 24, 6
    idx1, idx2, weights, biases, K, Bv = spec(rng, D, 16, 20, H, 2, K, scattered=True)
    weights[1] = np.eye(H, dtype=f32)
    biases[1] = np.zeros(H, f32)
    assert np.abs(biases[2]).min() > 0  # c_out nonzero: no sum of the row loop starts at a signed zero
    x = batch(rng, D, N)
    deep = layer(B, D, idx1, idx2, weights, biases, K, Bv, "leaky_relu", 0.0)
    nsf = B.Coupling(B.MLPSplineConditioner(weights[0], biases[0], weights[2], biases[2], K=K, B=Bv,
                                            activation="leaky_relu", slope=0.0), B.PartitionMask(D, idx1, idx2))
    run = lambda l: [B.to_numpy(a) for a in B.with_logabsdet_jacobian(B.inverse(l) if inv else l, B.from_numpy(x))]  # noqa: E731
    (yd, ld), (yn, ln) = run(deep), run(nsf)
    assert yd.tobytes() == yn.tobytes() and ld.tobytes() == ln.tobytes()


@pytest.mark.parametrize("inv", [False, True])
def test_slope_one_equals_the_spline_coupling(B, inv):
    """LeakyReLU(1) is the identity: the layer equals the device COUPLING_RQS layer on the product matrix, both within
    the gate of the float64 result.  W_out is scaled down so that the product network's raw knots stay moderate: with
    the spec's scale the log-Jacobians reach ±50 over 16 rows, and so steep a spline amplifies the rounding of the
    three layers in series beyond the reference's own float32 error."""
    rng = np.random.default_rng(5 + inv)
    D, N, K, Bv, M = 40, 3000, 6, 3.0, 3
    sp = spec(rng, D, 16, 20, 24, M, K, Bv, scattered=True)
    idx1, idx2, weights, biases = sp[:4]
    weights[-1] *= 0.25
    Wc, cc = weights[0].astype(np.float64), biases[0].astype(np.float64)
    for Wl, cl in zip(weights[1:], biases[1:]):
        Wc, cc = Wl @ Wc, Wl @ cc + cl
    x = batch(rng, D, N, Bv)
    deep = layer(B, D, *sp, "leaky_relu", 1.0)
    lin = B.Coupling(B.SplineConditioner(Wc.astype(f32), cc.astype(f32), K=K, B=Bv), B.PartitionMask(D, idx1, idx2))
    run = lambda l: [B.to_numpy(a) for a in B.with_logabsdet_jacobian(B.inverse(l) if inv else l, B.from_numpy(x))]  # noqa: E731
    (yn, ln), (yl, ll) = run(deep), run(lin)
    cols = list(range(0, N, 7))
    f = S.inverse if inv else S.forward
    y64, l64 = f(idx1, idx2, Wc, cc, K, Bv, x.astype(np.float64), cols=cols)
    y32, l32 = (DR.inverse if inv else DR.forward)(*sp, "leaky_relu", 1.0, x, f32, cols=cols)
    for y, l, what in ((yn, ln, "deep"), (yl, ll, "linear")):
        gate(y[:, cols], y64, y32, what + " y")
        gate(l[cols], l64, l32, what + " logjac")


def _raw(B, lay, inv, D, N, x, ldx, xoff, y, ldy, yoff, lj, acc):
    import torch

    from bijectors_jl_b200.interface import _desc_array

    arr = _desc_array(lay._descs(inv, D))
    L = B.lib()
    rc = L.b2b_chain_run_f32(arr, 1, ptr(x, xoff), ptr(y, yoff), ptr(lj), None, D, N, ldx, ldy, acc, None, 0, stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("M", [2, 3])
@pytest.mark.parametrize("inv", [False, True])
def test_layouts(B, inv, M):
    """Padded ld, misaligned bases, in place, accumulate and y == NULL give the bits of the plain call."""
    import torch

    rng = np.random.default_rng(11 + inv + M)
    D, N = 10, 333
    sp = spec(rng, D, 4, 3, 6, M, 5, scattered=True)
    x = batch(rng, D, N)
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
    assert _raw(B, lay, inv, D, N, xb, ld, 1, None, D, 0, lj, 0) == 0  # y == NULL
    assert lj.cpu().numpy().tobytes() == l0.tobytes()
    assert _raw(B, lay, inv, D, N, xb, ld, 1, xb, ld, 1, lj, 0) == 0  # in place
    assert xv[:, :D].cpu().numpy().T.tobytes() == y0.tobytes()
    assert (xv[:, D:] == sentinel).all() and lj.cpu().numpy().tobytes() == l0.tobytes()


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
@pytest.mark.parametrize("M", [2, 3, 4])
@pytest.mark.parametrize("D,n1,n2,H,K,N,with_c,cots", [
    (3, 1, 1, 1, 2, 300, True, "yl"), (10, 3, 4, 7, 5, 777, False, "yl"), (40, 20, 20, 33, 8, 1500, True, "y"),
    (64, 32, 32, 64, 8, 2000, True, "l"), (256, 128, 100, 128, 16, 150, True, "yl")])
def test_vjp(B, D, n1, n2, H, K, N, with_c, cots, M, act, slope, inv):
    import torch

    rng = np.random.default_rng(D + 3 * H + N + inv + 5 * M)
    sp = spec(rng, D, n1, n2, H, M, K, scattered=True, with_c=with_c)
    x = batch(rng, D, N)
    yb = rng.standard_normal((D, N)).astype(f32) if "y" in cots else None
    lb = rng.standard_normal(N).astype(f32) if "l" in cots else None
    lay = layer(B, D, *sp, act, slope)
    t = B.inverse(lay) if inv else lay
    xbar, grads = B.chain_vjp(t, B.from_numpy(x), None if yb is None else B.from_numpy(yb),
                              None if lb is None else torch.from_numpy(lb).cuda())
    xb64, g64 = DR.vjp(*sp, act, slope, x, yb, lb, inverse=inv)
    xb32, g32 = DR.vjp(*sp, act, slope, x, yb, lb, inverse=inv, dtype=f32)
    vjp_gate(B.to_numpy(xbar), xb64, xb32, "xbar", act)
    names = ("W_in", "W_hid", "W_out", "c") if with_c else ("W_in", "W_hid", "W_out")
    assert set(grads[0]) == set(names)
    for k in names:
        vjp_gate(grads[0][k].cpu().numpy(), g64[k], g32[k], k + "bar", act)


def _desc(B, D, n1, n2, H, M, K, act=0, with_c=True, inverse=0, Bv=3.0):
    import torch

    J = (3 * max(K, 1) - 1) * n1
    t = lambda n: torch.zeros((max(n, 1),), device="cuda")  # noqa: E731
    W_in, W_hid, W_out, c = t(H * n2), t((M - 1) * H * H), t(J * H), t(M * H + J)
    i1 = torch.arange(n1, dtype=torch.int32, device="cuda")
    i2 = torch.arange(n1, n1 + n2, dtype=torch.int32, device="cuda") % max(D, 1)
    d = B._lib.LayerDesc()
    d.kind, d.inverse = B._lib.COUPLING_DEEP_MLP_RQS, inverse
    d.n0, d.n1, d.n2, d.n3, d.f0, d.f1 = n1, n2, H, act | (K << 8) | (M << 16), 0.1, Bv
    d.p0, d.p1, d.p2, d.i0, d.i1 = W_in.data_ptr(), W_hid.data_ptr(), W_out.data_ptr(), i1.data_ptr(), i2.data_ptr()
    d.p3 = c.data_ptr() if with_c else None
    return d, (W_in, W_hid, W_out, c, i1, i2)


def test_cotangent_subsets(B):
    """Each requested subset of the four cotangents gets the oracle's values, the others stay untouched; both
    directions."""
    import itertools

    import torch

    from bijectors_jl_b200.interface import _desc_array

    rng = np.random.default_rng(23)
    D, N, M, K = 24, 900, 3, 5
    sp = spec(rng, D, 10, 12, 16, M, K, scattered=True)
    x = batch(rng, D, N)
    yb = rng.standard_normal((D, N)).astype(f32)
    lb = rng.standard_normal(N).astype(f32)
    L = B.lib()
    lay = layer(B, D, *sp)
    for inv in (False, True):
        xb64, g64 = DR.vjp(*sp, "tanh", 0.0, x, yb, lb, inverse=inv)
        xb32, g32 = DR.vjp(*sp, "tanh", 0.0, x, yb, lb, inverse=inv, dtype=f32)
        arr = _desc_array(lay._descs(inv, D))
        xd, ybd = B.from_numpy(x), B.from_numpy(yb)
        lbd = torch.from_numpy(lb).cuda()
        wsb = L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
        ws = torch.empty((max(wsb, 1),), dtype=torch.uint8, device="cuda")
        shapes = [g64[k].size for k in ("W_in", "W_hid", "W_out", "c")]
        for sub in itertools.chain.from_iterable(itertools.combinations(range(4), r) for r in (1, 2, 4)):
            bars = [torch.full((n,), 9.5, device="cuda") if i in sub else None for i, n in enumerate(shapes)]
            ptrs = (ctypes.c_void_p * 4)(*[None if b is None else b.data_ptr() for b in bars])
            xbar = B.colmajor_empty(D, N, "cuda")
            rc = L.b2b_chain_vjp_f32(arr, 1, xd.data_ptr(), ybd.data_ptr(), lbd.data_ptr(), xbar.data_ptr(),
                                     ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), wsb, stream())
            assert rc == 0
            torch.cuda.synchronize()
            vjp_gate(B.to_numpy(xbar), xb64, xb32, ("xbar", sub))
            for i, k in enumerate(("W_in", "W_hid", "W_out", "c")):
                if i in sub:
                    # device storage is column-major per matrix: compare against the transpose of each matrix
                    got = bars[i].cpu().numpy()
                    want64, want32 = g64[k], g32[k]
                    if k == "W_hid":
                        want64, want32 = want64.transpose(0, 2, 1), want32.transpose(0, 2, 1)
                    elif k != "c":
                        want64, want32 = want64.T, want32.T
                    vjp_gate(got, want64.ravel(), want32.ravel(), (k, sub, inv))


def test_envelope_corner_vjp(B):
    """n1 = n2 = H = 128, K = 16, M = 4 at D = 1024: the largest shared-memory footprint of the reverse kernel."""
    import torch

    rng = np.random.default_rng(29)
    D, N, M, K = 1024, 130, 4, 16
    sp = spec(rng, D, 128, 128, 128, M, K, scattered=True)
    x = batch(rng, D, N)
    yb = rng.standard_normal((D, N)).astype(f32)
    lb = rng.standard_normal(N).astype(f32)
    lay = layer(B, D, *sp)
    for inv in (False, True):
        xbar, grads = B.chain_vjp(B.inverse(lay) if inv else lay, B.from_numpy(x), B.from_numpy(yb),
                                  torch.from_numpy(lb).cuda())
        xb64, g64 = DR.vjp(*sp, "tanh", 0.0, x, yb, lb, inverse=inv)
        xb32, g32 = DR.vjp(*sp, "tanh", 0.0, x, yb, lb, inverse=inv, dtype=f32)
        vjp_gate(B.to_numpy(xbar), xb64, xb32, "xbar")
        for k in ("W_in", "W_hid", "W_out", "c"):
            vjp_gate(grads[0][k].cpu().numpy(), g64[k], g32[k], (k, inv))


@pytest.mark.parametrize("D,n1,n2,H,M,K,act,want", [(300, 129, 1, 4, 2, 4, 0, -2), (300, 1, 129, 4, 2, 4, 0, -2),
                                                    (40, 4, 4, 129, 2, 4, 0, -2), (40, 4, 4, 4, 5, 4, 0, -2),
                                                    (40, 4, 4, 4, 2, 17, 1, -2), (1025, 4, 4, 4, 3, 4, 1, -2),
                                                    (40, 4, 4, 4, 2, 4, 2, -1), (40, 4, 4, 4, 1, 4, 0, -1)])
def test_refused_with_nothing_launched(B, D, n1, n2, H, M, K, act, want):
    import torch

    L = B.lib()
    N = 100
    d, keep = _desc(B, D, n1, n2, H, M, K, act)
    arr = (B._lib.LayerDesc * 1)(d)
    x = torch.zeros((N * D,), device="cuda")
    y = torch.full((N * D,), 3.5, device="cuda")
    lj = torch.full((N,), 3.5, device="cuda")
    xb = torch.full((N * D,), 3.5, device="cuda")
    torch.cuda.synchronize()
    if want == -2:
        assert L.b2b_chain_workspace_bytes(arr, 1, D, N, 1, 0) == 0
    assert L.b2b_chain_vjp_workspace_bytes(arr, 1, D, N) == 0
    assert L.b2b_chain_run_f32(arr, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream()) == want
    assert L.b2b_last_launch_count() == 0
    assert L.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, None, 0, stream()) == want
    assert L.b2b_last_launch_count() == 0
    torch.cuda.synchronize()
    assert (y == 3.5).all() and (lj == 3.5).all() and (xb == 3.5).all()


def _flow(B, rng, D, H=12):
    """Planar ∘ deep neural spline coupling (M = 2, LeakyReLU) ∘ Permute ∘ deep affine coupling ∘ BatchNorm ∘ neural
    spline coupling ∘ deep neural spline coupling (M = 3, tanh), in application order from the right."""
    dev, ora = [], []
    sp = spec(rng, D, D // 2, D - D // 2, H, 3, 6)
    dev.append(layer(B, D, *sp))
    ora.append(DR.DeepMLPSplineLayer(*sp))
    i1, i2 = list(range(1, D // 3 + 1)), list(range(D // 3 + 1, D + 1))
    W1 = (rng.standard_normal((H, len(i2))) * 0.3).astype(f32)
    W2 = (rng.standard_normal((17 * len(i1), H)) * 0.2).astype(f32)
    c1, c2 = (rng.standard_normal(H) * 0.1).astype(f32), (rng.standard_normal(17 * len(i1)) * 0.1).astype(f32)
    dev.append(B.Coupling(B.MLPSplineConditioner(W1, c1, W2, c2, K=6, B=3.0), B.PartitionMask(D, i1, i2)))
    ora.append(R.MLPSplineLayer(i1, i2, W1, c1, W2, c2, 6, 3.0))
    b, logs = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
    m, v = (rng.standard_normal(D) * 0.1).astype(f32), (rng.uniform(0.5, 1.5, D)).astype(f32)
    dev.append(B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v))
    ora.append(O.Layer("batchnorm", dict(bn=O.BatchNormParams(b=b, logs=logs, m=m, v=v, eps=1e-5))))
    j1, j2 = list(range(D // 2 + 1, D + 1)), list(range(1, D // 2 + 1))
    Ws = [(rng.standard_normal((H, len(j2))) * 0.3).astype(f32), (rng.standard_normal((H, H)) * 0.3).astype(f32),
          (rng.standard_normal((2 * len(j1), H)) * 0.1).astype(f32)]
    dev.append(B.Coupling(B.DeepMLPConditioner(Ws), B.PartitionMask(D, j1, j2)))
    ora.append(DM.DeepMLPLayer(j1, j2, Ws))
    perm = rng.permutation(D) + 1
    dev.append(B.Permute(perm))
    ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))))
    sp = spec(rng, D, D // 3, D - D // 3 - 1, H + 1, 2, 4, scattered=True)
    dev.append(layer(B, D, *sp, "leaky_relu", 0.2))
    ora.append(DR.DeepMLPSplineLayer(*sp, "leaky_relu", 0.2))
    w, u = (rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32)
    bb = rng.standard_normal(1).astype(f32)
    dev.append(B.PlanarLayer(w, u, bb))
    ora.append(O.Layer("planar", dict(w=w, u=u, b=bb)))
    return B.Composed(*dev), ora


DEEP_AT = (0, 5)  # flow positions of the deep spline couplings
NAMES = ("W_in", "W_hid", "W_out", "c")


@pytest.mark.parametrize("base", ["diag", "tril"])
def test_chain_logpdf_and_vjp(B, base):
    import torch

    rng = np.random.default_rng(31 + (base == "tril"))
    D, N = 16, 600
    flow, ora = _flow(B, rng, D)
    y = rng.standard_normal((D, N)).astype(f32)
    mu = (rng.standard_normal(D) * 0.2).astype(f32)
    if base == "diag":
        sigma = rng.uniform(0.7, 1.3, D).astype(f32)
        dist, kw = B.MvNormal(D, mu=mu, sigma=sigma), dict(mu=mu, sigma=sigma, terminal=True)
    else:
        L = T.random_tril(rng, D).astype(f32)
        dist, kw = B.MvNormal(D, mu=mu, scale_tril=L), dict(mu=mu, scale_tril=L)
    td = B.transformed(dist, flow)
    yd = B.from_numpy(y)
    lp = B.to_numpy(B.logpdf(td, yd))
    inv_layers, flags = ora[::-1], [True] * len(ora)
    _, lp64 = V.chain_logjac(inv_layers, flags, y.astype(np.float64), **kw)
    _, lp32 = V.chain_logjac(inv_layers, flags, y, dtype=f32, **kw)
    gate(lp, lp64, lp32, "logpdf")
    s, lps = B.logpdf_sum(td, yd)
    assert B.to_numpy(lps).tobytes() == lp.tobytes()
    assert abs(float(s) - lp64.sum()) <= max(1e-5, 2 * abs(lp32.sum(dtype=np.float64) - lp64.sum())) * abs(lp64.sum()) + 1e-3
    lb = rng.standard_normal(N).astype(f32)
    ybar, fgrads, _ = B.logpdf_vjp(td, yd, torch.from_numpy(lb).cuda())
    g64, grads64, _ = V.chain_vjp(inv_layers, flags, y.astype(np.float64), None, lb, **kw)
    g32, grads32, _ = V.chain_vjp(inv_layers, flags, y, None, lb, dtype=f32, **kw)
    chain_gate(B.to_numpy(ybar), g64, g32, "ybar")
    for k in DEEP_AT:  # flow order; the oracle's list is in application order of the inverse chain
        for name in NAMES:
            chain_gate(fgrads[k][name].cpu().numpy(), grads64[::-1][k][name], grads32[::-1][k][name], (k, name))
    # chain_vjp of the forward flow
    x = rng.standard_normal((D, N)).astype(f32)
    ybf = rng.standard_normal((D, N)).astype(f32)
    xbar, cg = B.chain_vjp(flow, B.from_numpy(x), B.from_numpy(ybf), torch.from_numpy(lb).cuda())
    fl = [False] * len(ora)
    x64, c64, _ = V.chain_vjp(ora, fl, x.astype(np.float64), ybf, lb)
    x32, c32, _ = V.chain_vjp(ora, fl, x, ybf, lb, dtype=f32)
    chain_gate(B.to_numpy(xbar), x64, x32, "xbar")
    for k in DEEP_AT:
        for name in NAMES:
            chain_gate(cg[k][name].cpu().numpy(), c64[k][name], c32[k][name], ("fwd", k, name))


def test_rand_and_host_path(B):
    rng = np.random.default_rng(41)
    D, N = 16, 3001
    flow, ora = _flow(B, rng, D)
    td = B.transformed(B.MvNormal(D), flow)
    y, lj = B.rand(td, N, seed=77, offset=2, with_logjac=True)
    x = B.rand(td.dist, N, seed=77, offset=2)
    y2, lj2 = B.run_chain(flow, x)
    assert B.to_numpy(y).tobytes() == B.to_numpy(y2).tobytes() and B.to_numpy(lj).tobytes() == B.to_numpy(lj2).tobytes()
    z = O.philox_normals(77, 2, D, N)[:, :300]
    y64, l64 = O.chain_forward(ora, z.astype(np.float64))
    y32, l32 = O.chain_forward(ora, z.astype(f32))
    gate(B.to_numpy(y)[:, :300], y64, y32, "rand y")
    gate(B.to_numpy(lj)[:300], l64, l32, "rand logjac")
    xh = B.from_numpy(B.to_numpy(x), device="cpu")
    yh, ljh = B.run_chain(flow, xh)
    assert B.to_numpy(yh).tobytes() == B.to_numpy(y2).tobytes()
    assert B.to_numpy(ljh).tobytes() == B.to_numpy(lj2).tobytes()


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
    e = B.colmajor_empty(D, 0, "cuda")
    _, ge = B.chain_vjp(flow, e)
    assert all(float(t.abs().sum()) == 0 for gg in ge for t in gg.values())


def test_training_lowers_nll_and_first_gradient(B):
    """Three deep neural spline couplings with permutations over an MvNormal base at D = 8, trained with Adam on
    seeded data: the first gradient of every parameter matches the float64 oracle and the NLL goes down."""
    import torch

    rng = np.random.default_rng(81)
    D, N, H, K, Bv = 8, 4096, 16, 6, 4.0
    blocks, ora = [], []
    for k in range(3):
        i1, i2 = list(range(1, D // 2 + 1)), list(range(D // 2 + 1, D + 1))
        M = 2 + k
        J = (3 * K - 1) * len(i1)
        Ws = [(rng.standard_normal((H, len(i2))) * 0.3).astype(f32)]
        Ws += [(rng.standard_normal((H, H)) * 0.3).astype(f32) for _ in range(M - 1)]
        Ws += [(rng.standard_normal((J, H)) * 0.05).astype(f32)]
        bs = [(rng.standard_normal(H) * 0.1).astype(f32) for _ in range(M)] + [np.zeros(J, f32)]
        act = ("tanh", 0.0) if k % 2 == 0 else ("leaky_relu", 0.1)
        blocks.append(layer(B, D, i1, i2, Ws, bs, K, Bv, *act))
        ora.append(DR.DeepMLPSplineLayer(i1, i2, Ws, bs, K, Bv, *act))
        perm = np.roll(np.arange(1, D + 1), 3)
        blocks.append(B.Permute(perm))
        ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))))
    flow = B.autograd.Flow(B.Composed(*blocks))
    assert len(flow.params) == 12
    z = rng.standard_normal((D, N))
    data = np.stack([z[0] * 1.5, z[1] * 0.5 + 0.3 * z[0] ** 2] + [z[j] * (0.5 + 0.1 * j) for j in range(2, D)]).astype(f32)
    y = B.from_numpy(data)
    nll = flow.nll(y)
    nll.backward()
    inv_layers, flags = ora[::-1], [True] * len(ora)
    _, lp = V.chain_logjac(inv_layers, flags, data.astype(np.float64), mu=None, sigma=None, terminal=True)
    assert abs(float(nll) + lp.sum()) <= 1e-4 * abs(lp.sum())
    lb = -np.ones(N)
    _, g64, _ = V.chain_vjp(inv_layers, flags, data.astype(np.float64), None, lb, mu=None, sigma=None, terminal=True)
    _, g32, _ = V.chain_vjp(inv_layers, flags, data, None, lb.astype(f32), mu=None, sigma=None, terminal=True, dtype=f32)
    g64, g32 = g64[::-1], g32[::-1]  # flow order
    for k in range(3):
        for i, name in enumerate(NAMES):
            got = flow.params[4 * k + i].grad.cpu().numpy()
            if got.ndim == 2:
                got = got.T
            elif got.ndim == 3:
                got = got.transpose(0, 2, 1)
            chain_gate(got, g64[2 * k][name], g32[2 * k][name], (k, name))
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    first = float(nll)
    for _ in range(30):
        opt.zero_grad()
        loss = flow.nll(y)
        loss.backward()
        opt.step()
    assert float(flow.nll(y)) < first - 0.02 * abs(first)


@pytest.mark.parametrize("inv", [False, True])
def test_periodic_training_batch(B, inv):
    """N ≈ 2²⁰ columns repeating 4099: every column of x̄ and the four parameter cotangents against q·P(period) + P(rest)
    in float64, as test_coupling_mlp_rqs.py checks kind 14.  The x̄ gate's XRTOL is 16× and XFLOOR 4× (kind 14: 2×
    both): x̄₂ passes through the M + 1 GEMMs of the network in series, each in the device's fixed fmaf order, and on
    the steepest columns of the inverse case (‖x̄ₙ‖ ≈ 5× the rms) the device's error reached 1.2e-4 of the column's
    norm, 6.5× the float32 reference's own."""
    import torch

    N, Mc = TB.N_MLP, TB.M
    N = min(N, (1 << 20) + 13)
    rng = np.random.default_rng(91 + inv)
    D = 64
    sp = spec(rng, D, 24, 40, 32, 3, 8, scattered=True) if inv else spec(rng, D, 32, 32, 64, 2, 8)
    TB._need_memory(3 * D * N * 4 + N * 4 * 16)
    q, r = divmod(N, Mc)
    X = MC.inputs(rng, D, Mc)
    Y = rng.standard_normal((D, Mc)).astype(f32)
    Lb = rng.standard_normal(Mc).astype(f32)
    lay = layer(B, D, *sp)
    xbar, grads = B.chain_vjp(B.inverse(lay) if inv else lay, TB._periodic(X, N, f32), TB._periodic(Y, N, f32),
                              TB._periodic(Lb, N, f32))
    torch.cuda.synchronize()
    o64 = DR.vjp(*sp, "tanh", 0.0, X.astype(np.float64), Y, Lb, inverse=inv)
    o32 = DR.vjp(*sp, "tanh", 0.0, X, Y, Lb, inverse=inv, dtype=f32)
    o64r = DR.vjp(*sp, "tanh", 0.0, X[:, :r].astype(np.float64), Y[:, :r], Lb[:r], inverse=inv)
    TB.check_columns(xbar, np.asarray(o64[0]), np.asarray(o32[0]), rtol=16 * TB.XRTOL, floor=4 * TB.XFLOOR,
                     what=f"deep nsf inv={inv}")
    for k in NAMES:
        d = np.asarray(grads[0][k].cpu().numpy(), np.float64).ravel()  # in the parameter's orientation
        ref = (q * o64[1][k] + o64r[1][k]).ravel()
        tol = max(TB.PRTOL, 4 * rel(o32[1][k], o64[1][k]))
        assert rel(d, ref) <= tol, (k, rel(d, ref), tol)
