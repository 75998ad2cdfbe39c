"""GPU tests of chains that mix every layer kind -- own-launch kinds (spline / MLP / affine coupling, dense Scale, the TRIL
terminal) back to back with fused runs -- against the float64 chain reference of tests/chain_vjp_oracle.py: forward,
inverse, layouts, logpdf and its batch sum, reverse mode and the training path.  These chains route every segment of the
chain orchestration: launches reading y in place after another own launch, the D x N scratch when y == NULL, BatchNorm
folded before and after a coupling, planar runs embedded at Dk != D between own launches, and both parities of the
cotangent ping-pong.  Gates are tied to the reference's own float32 error on the same input, as in test_gpu_parity:
max(1e-5, 2 × ‖oracle32 − oracle64‖ / ‖oracle64‖), norm-wise."""
import ctypes

import numpy as np
import pytest

import chain_vjp_oracle as V
import coupling_mlp_oracle as M
import mvnormal_tril_oracle as T
import scale_matrix_oracle as SM
import spline_coupling_oracle as SC
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5
EW = O.EW


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(dev, a64, a32, what="", floor=RTOL, k=2.0):
    tol = max(floor, k * rel(a32, a64))
    e = rel(dev, a64)
    assert e <= tol, (what, e, tol)


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def stream():
    import torch

    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- the chains -------------------------------------------------------------------------------------------------------------
def _rows(rng, D, n1, n2, lists):
    rows = (rng.permutation(D) if lists else np.arange(D)) + 1
    return [int(i) for i in rows[:n1]], [int(i) for i in rows[n1:n1 + n2]]


def _layer(B, rng, D, kind, o):
    """(device layer, oracle layer) of one chain element."""
    if kind == "stacked":
        k = D // 3
        ranges = [(1, k), (k + 1, 2 * k), (2 * k + 1, D)]
        return (B.Stacked([B.Shift(0.3), B.Scale(-1.2), B.LeakyReLU(0.5)], ranges),
                O.Layer("stacked", dict(ops=[(EW.SHIFT, f32(0.3)), (EW.SCALE, f32(-1.2)), (EW.LEAKY_RELU, f32(0.5))],
                                        ranges=ranges)))
    if kind == "perm":
        perm = (rng.permutation(D) + 1).tolist()
        return B.Permute(perm), O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm)))
    if kind == "rqs":
        K = 8
        spl = B.RationalQuadraticSpline(*(rng.standard_normal(s).astype(f32) * 0.5 for s in ((D, K), (D, K), (D, K - 1))),
                                        3.0)
        W, H, Dv = spl.knots()
        return spl, O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv))
    if kind == "bn":
        b, logs, m = ((rng.standard_normal(D) * 0.1).astype(f32) for _ in range(3))
        v = rng.uniform(0.5, 1.5, D).astype(f32)
        return (B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v),
                O.Layer("batchnorm", dict(bn=O.BatchNormParams(b, logs, m, v, f32(1e-5), f32(0.1)))))
    if kind == "cpl":
        i1, i2 = _rows(rng, D, o["n1"], o["n2"], o.get("lists", False))
        W = (rng.standard_normal((2 * len(i1), len(i2))) * 0.1 / np.sqrt(len(i2))).astype(f32)
        c = (rng.standard_normal(2 * len(i1)) * 0.1).astype(f32)
        return (B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, i1, i2)),
                O.Layer("coupling_affine", dict(idx1=np.asarray(i1), idx2=np.asarray(i2), W=W, c=c)))
    if kind == "spl":
        K = o.get("K", 8)
        i1, i2 = _rows(rng, D, o["n1"], o["n2"], o.get("lists", True))
        W = (rng.standard_normal(((3 * K - 1) * len(i1), len(i2))) * 0.3 / np.sqrt(len(i2))).astype(f32)
        c = (rng.standard_normal((3 * K - 1) * len(i1)) * 0.3).astype(f32)
        return (B.Coupling(B.SplineConditioner(W, c, K=K, B=3.0), B.PartitionMask(D, i1, i2)),
                SC.SplineLayer(i1, i2, W, c, K, 3.0))
    if kind == "scale":
        A = SM.well_conditioned(rng, D).astype(f32)
        return B.Scale(A), SM.ScaleLayer(A)
    if kind == "mlp":
        i1, i2 = _rows(rng, D, o["n1"], o["n2"], o.get("lists", True))
        H, act, slope = o["H"], o.get("act", "tanh"), o.get("slope", 0.0)
        W1 = (rng.standard_normal((H, len(i2))) * 0.8 / np.sqrt(len(i2))).astype(f32)
        W2 = (rng.standard_normal((2 * len(i1), H)) * 0.3 / np.sqrt(H)).astype(f32)
        c1, c2 = (rng.standard_normal(H) * 0.3).astype(f32), (rng.standard_normal(2 * len(i1)) * 0.1).astype(f32)
        return (B.Coupling(B.MLPConditioner(W1, c1, W2, c2, activation=act, slope=slope), B.PartitionMask(D, i1, i2)),
                M.MLPLayer(i1, i2, W1, c1, W2, c2, act, slope))
    if kind == "planar":
        w, u = ((rng.standard_normal(D) * 0.3 / np.sqrt(D)).astype(f32) for _ in range(2))
        b = rng.standard_normal(1).astype(f32)
        return B.PlanarLayer(w, u, b), O.Layer("planar", dict(w=w, u=u, b=b))
    if kind == "radial":
        a, be = rng.standard_normal(1).astype(f32), rng.standard_normal(1).astype(f32)
        z0 = (rng.standard_normal(D) * 0.1).astype(f32)
        return B.RadialLayer(a, be, z0), O.Layer("radial", dict(alpha_raw=a, beta=be, z0=z0))
    raise ValueError(kind)


def _long24():
    own = [("spl", 0, dict(n1=12, n2=20)), ("mlp", 1, dict(n1=16, n2=16, H=24)), ("scale", 0, {}),
           ("cpl", 0, dict(n1=10, n2=14, lists=True)), ("mlp", 0, dict(n1=8, n2=20, H=16, act="leaky_relu", slope=0.1)),
           ("spl", 1, dict(n1=16, n2=16, K=4)), ("scale", 1, {}), ("cpl", 1, dict(n1=16, n2=16))]
    fused = [("planar", 0, {}), ("stacked", 0, {}), ("radial", 1, {}), ("bn", 0, {}), ("perm", 0, {}), ("planar", 1, {}),
             ("rqs", 0, {}), ("radial", 0, {})]
    out = []
    for k in range(12):
        out += [own[k % 8], fused[k % 8]]
    return out[:23]


# name: (D, [(kind, inverse, options)], bases of the logpdf tests)
CHAINS = {
    "every64": (64, [("stacked", 0, {}), ("perm", 0, {}), ("rqs", 0, {}), ("bn", 0, {}), ("cpl", 0, dict(n1=32, n2=32)),
                     ("bn", 1, {}), ("spl", 0, dict(n1=16, n2=24)), ("scale", 0, {}), ("mlp", 0, dict(n1=20, n2=24, H=32)),
                     ("mlp", 1, dict(n1=24, n2=20, H=16, act="leaky_relu", slope=0.2)), ("planar", 0, {}),
                     ("planar", 1, {}), ("planar", 0, {}), ("radial", 0, {}), ("radial", 1, {})], ("diag", "tril")),
    "scale-spl-planar-mlp20": (20, [("scale", 0, {}), ("spl", 0, dict(n1=8, n2=12)), ("planar", 0, {}),
                                    ("mlp", 0, dict(n1=10, n2=10, H=16))], ("tril",)),
    "inverse100": (100, [("mlp", 1, dict(n1=40, n2=60, H=48)), ("planar", 1, {}), ("planar", 1, {}), ("planar", 1, {}),
                         ("planar", 1, {}), ("scale", 1, {}), ("spl", 1, dict(n1=50, n2=50))], ("diag",)),
    "envelope256": (256, [("bn", 0, {}), ("cpl", 0, dict(n1=128, n2=128)), ("bn", 0, {}),
                          ("spl", 0, dict(n1=128, n2=128, K=16, lists=False)), ("scale", 0, {}),
                          ("mlp", 0, dict(n1=128, n2=128, H=256, lists=False))], ("tril",)),
    "wide1024": (1024, [("stacked", 0, {}), ("spl", 0, dict(n1=128, n2=128)), ("mlp", 0, dict(n1=128, n2=128, H=64)),
                        ("cpl", 0, dict(n1=100, n2=128, lists=True)), ("bn", 0, {})], ("diag",)),
    "long32": (32, _long24(), ("diag",)),
}


def build(B, name, seed=0):
    """(D, device layers, oracle layers, inverse flags) of CHAINS[name] (device layer l is inverted when flags[l])."""
    D, spec, _ = CHAINS[name]
    rng = np.random.default_rng(len(name) * 1000 + D + seed)
    dev, ora, flags = [], [], []
    for kind, inv, o in spec:
        d, r = _layer(B, rng, D, kind, o)
        dev.append(B.inverse(d) if inv else d)
        ora.append(r)
        flags.append(bool(inv))
    return D, dev, ora, flags


def inputs(rng, D, N):
    return (rng.standard_normal((D, N)) * 0.7).astype(f32)


def base_of(B, rng, D, kind):
    """(device MvNormal, oracle keywords of V.chain_logjac / chain_vjp)."""
    mu = (rng.standard_normal(D) * 0.2).astype(f32)
    if kind == "diag":
        sigma = rng.uniform(0.7, 1.4, D).astype(f32)
        return B.MvNormal(D, mu=mu, sigma=sigma), dict(mu=mu, sigma=sigma, terminal=True)
    L = T.random_tril(rng, D).astype(f32)
    return B.MvNormal(D, mu=mu, scale_tril=L), dict(mu=mu, scale_tril=L)


def inverted(ora, flags):
    return ora[::-1], [not f for f in flags[::-1]]


BASES = [(name, b) for name, (_, _, bases) in CHAINS.items() for b in bases]


# ---- forward and inverse ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 7, 1501, 65539])
@pytest.mark.parametrize("name", list(CHAINS))
def test_forward_inverse(B, name, N):
    D, dev, ora, flags = build(B, name)
    rng = np.random.default_rng(N + D)
    x = inputs(rng, D, N)
    flow = B.Composed(*dev)
    y, lj = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(flow, B.from_numpy(x)))
    xr, ljr = (B.to_numpy(a) for a in B.with_logabsdet_jacobian(B.inverse(flow), B.from_numpy(y)))
    assert np.isfinite(y).all() and np.isfinite(lj).all() and np.isfinite(xr).all()
    sel = slice(None) if N <= 5000 else np.unique(np.r_[0, 1, N - 1, rng.integers(0, N, 300)])
    y64, l64 = V.chain_logjac(ora, flags, x[:, sel].astype(np.float64))
    y32, l32 = V.chain_logjac(ora, flags, x[:, sel], dtype=f32)
    gate(y[:, sel], y64, y32, "y")
    gate(lj[sel], l64, l32, "logjac")
    io, iflags = inverted(ora, flags)
    x64, li64 = V.chain_logjac(io, iflags, y[:, sel].astype(np.float64))
    x32, li32 = V.chain_logjac(io, iflags, y[:, sel], dtype=f32)
    gate(xr[:, sel], x64, x32, "x")
    gate(ljr[sel], li64, li32, "inverse logjac")


# ---- layouts: bit for bit against the dense call --------------------------------------------------------------------------
def _run(B, arr, L, D, N, x, ldx, y, ldy, lj, acc, sum_out=None, want_sum=0, fill=None):
    import torch

    lib = B.lib()
    ws_b = lib.b2b_chain_workspace_bytes(arr, L, D, N, int(y is not None), want_sum)
    ws = torch.empty(max(ws_b, 4), dtype=torch.uint8, device="cuda")
    if fill is not None:
        ws.view(torch.float32)[: ws.numel() // 4].fill_(fill)
    p = lambda t: None if t is None else t  # noqa: E731
    rc = lib.b2b_chain_run_f32(arr, L, x, p(y), p(lj), p(sum_out), D, N, ldx, ldy, acc, ws.data_ptr(), ws_b, stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("name", list(CHAINS))
def test_layouts(B, name):
    D, dev, _, _ = build(B, name)
    N = 1031
    # one kernel per launch for every call (the fp32 CUDA-core coupling kernel, the lane-group fused kernel): the
    # tensor-core coupling and TMA-staged fused kernels take only aligned operands, so a strided call would otherwise
    # round differently from the dense one by design
    assert B.lib().b2b_set_kernel_variant(11) == 0
    try:
        _layouts(B, D, dev, N)
    finally:
        B.lib().b2b_set_kernel_variant(0)


def _layouts(B, D, dev, N):
    import torch

    from bijectors_jl_b200.interface import _desc_array

    rng = np.random.default_rng(D + 5)
    x = inputs(rng, D, N)
    descs = B.Composed(*dev)._descs(False, D)
    arr, L = _desc_array(descs), len(descs)
    xd = B.from_numpy(x)
    y0 = B.colmajor_empty(D, N)
    l0 = torch.empty(N, device="cuda")
    assert _run(B, arr, L, D, N, xd.data_ptr(), D, y0.data_ptr(), D, l0.data_ptr(), 0) == 0
    y0, l0 = B.to_numpy(y0), l0.cpu().numpy()
    sentinel = 7.25
    ldx, ldy = D + 3, D + 5
    xb = torch.full((ldx * N + 8,), sentinel, device="cuda")
    xv = xb[1:1 + ldx * N].view(N, ldx)
    xv[:, :D] = torch.from_numpy(x.T.copy()).cuda()
    yb = torch.full((ldy * N + 8,), sentinel, device="cuda")
    yv = yb[3:3 + ldy * N].view(N, ldy)
    lj = torch.empty(N, device="cuda")
    assert _run(B, arr, L, D, N, xv.data_ptr(), ldx, yv.data_ptr(), ldy, lj.data_ptr(), 0) == 0
    assert yv[:, :D].cpu().numpy().T.tobytes() == y0.tobytes()
    assert (yv[:, D:] == sentinel).all() and (yb[:3] == sentinel).all() and (yb[3 + ldy * N:] == sentinel).all()
    assert lj.cpu().numpy().tobytes() == l0.tobytes()
    assert (xv[:, D:] == sentinel).all() and xv[:, :D].cpu().numpy().T.tobytes() == x.tobytes()  # x untouched
    base = torch.randn(N, device="cuda")
    lj.copy_(base)
    assert _run(B, arr, L, D, N, xv.data_ptr(), ldx, yv.data_ptr(), ldy, lj.data_ptr(), 1) == 0  # accumulate
    want = base.cpu().numpy() + l0
    assert rel(lj.cpu().numpy(), want) <= 1e-6  # the per-launch order of additions differs from base + Σ
    lj.fill_(float("nan"))
    assert _run(B, arr, L, D, N, xv.data_ptr(), ldx, None, D, lj.data_ptr(), 0, fill=float("nan")) == 0  # y == NULL
    assert lj.cpu().numpy().tobytes() == l0.tobytes()
    lj.fill_(float("nan"))
    assert _run(B, arr, L, D, N, xv.data_ptr(), ldx, xv.data_ptr(), ldx, lj.data_ptr(), 0) == 0  # y == x
    assert xv[:, :D].cpu().numpy().T.tobytes() == y0.tobytes() and (xv[:, D:] == sentinel).all()
    assert lj.cpu().numpy().tobytes() == l0.tobytes()


# ---- logpdf and its batch sum ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,base", BASES)
def test_logpdf_and_batch_sum(B, name, base):
    """logpdf, logpdf_sum and the raw batch sum without logjac (accumulate_logjac 0 and 1, workspace full of NaN): the
    sums agree bit for bit and match the float64 Σ; a chain of several launches must carry every launch's log-Jacobian
    into the sum."""
    import torch

    from bijectors_jl_b200.interface import _desc_array

    D, dev, ora, flags = build(B, name)
    rng = np.random.default_rng(D + 11 + len(base))
    N = 1501
    x = inputs(rng, D, N)
    bd, kw = base_of(B, rng, D, base)
    td = B.transformed(bd, B.inverse(B.Composed(*dev)))  # logpdf runs the chain itself, then the base
    xd = B.from_numpy(x)
    lp = B.to_numpy(B.logpdf(td, xd))
    _, lp64 = V.chain_logjac(ora, flags, x.astype(np.float64), **kw)
    _, lp32 = V.chain_logjac(ora, flags, x, dtype=f32, **kw)
    gate(lp, lp64, lp32, "logpdf")
    s, lps = B.logpdf_sum(td, xd)
    assert B.to_numpy(lps).tobytes() == lp.tobytes()
    s = float(s)
    assert abs(s - float(np.sum(lp, dtype=np.float64))) <= 1e-9 * abs(s)
    s64, s32 = float(lp64.sum()), float(np.sum(lp32, dtype=np.float64))
    assert abs(s - s64) <= max(RTOL, 2 * abs(s32 - s64) / abs(s64)) * abs(s64)
    descs = list(B.Composed(*dev)._descs(False, D)) + [bd._terminal_desc()]
    arr, L = _desc_array(descs), len(descs)
    out = torch.empty((), dtype=torch.float64, device="cuda")
    for acc in (0, 1):
        out.fill_(float("nan"))
        assert _run(B, arr, L, D, N, xd.data_ptr(), D, None, D, None, acc, out.data_ptr(), 1, fill=float("nan")) == 0
        assert float(out) == s, (acc, float(out), s)


@pytest.mark.parametrize("kind", ["cpl", "mlp"])
def test_batch_sum_without_logjac_two_launches(B, kind):
    """[coupling, MVNORMAL_DIAG] and [MLP coupling, Stacked, MVNORMAL_DIAG]: the smallest chains whose batch sum without
    logjac crosses a launch boundary."""
    import torch

    from bijectors_jl_b200.interface import _desc_array

    rng = np.random.default_rng(7 + len(kind))
    D, N = 32, 4099
    spec = [("cpl", 0, dict(n1=16, n2=16))] if kind == "cpl" else [("mlp", 0, dict(n1=16, n2=16, H=32)), ("stacked", 0, {})]
    dev, ora = zip(*[_layer(B, rng, D, k, o) for k, _, o in spec])
    bd, kw = base_of(B, rng, D, "diag")
    x = inputs(rng, D, N)
    descs = list(B.Composed(*dev)._descs(False, D)) + [bd._terminal_desc()]
    arr, L = _desc_array(descs), len(descs)
    out = torch.empty((), dtype=torch.float64, device="cuda")
    assert _run(B, arr, L, D, N, B.from_numpy(x).data_ptr(), D, None, D, None, 0, out.data_ptr(), 1, fill=float("nan")) == 0
    s64 = float(V.chain_logjac(list(ora), [False] * len(ora), x.astype(np.float64), **kw)[1].sum())
    assert abs(float(out) - s64) <= 1e-5 * abs(s64), (float(out), s64)


# ---- reverse mode -------------------------------------------------------------------------------------------------------------
def _strided(B, a, off, ld):
    """A (D, N) device batch at a float offset `off` with leading dimension `ld` (padding rows hold NaN)."""
    import torch

    D, N = a.shape
    buf = torch.full((ld * N + off + 8,), float("nan"), device="cuda")
    v = buf[off:off + ld * N].view(N, ld)
    v[:, :D] = torch.from_numpy(np.ascontiguousarray(a.T)).cuda()
    return v[:, :D].t()


# The gate of reverse mode is max(3e-4, 4 × the float32 reference's own error).  Each segment's VJP alone matches float64
# to ~1e-7 here, but the chain's inputs to a spline coupling are recomputed in float32 on the device and the coupling's
# VJP is sensitive to them (alone, on one float32 input, one of the 23-layer chain's spline couplings is ~2e-5 off float64
# on x̄, device and float32 reference alike); the float32 reference rounds those inputs differently, so its own error
# does not bound the device's.  Through the 23-layer chain that reaches ~2e-4 on x̄ and the parameter cotangents before it.  A wrong slot,
# checkpoint or cotangent buffer is off by O(1).
VJP_FLOOR = 3e-4


def check_vjp(B, dev_t, ora, flags, x, ybar, lb, kw=None, bd=None, layout="dense"):
    """chain_vjp / logpdf_vjp against the reference: x̄, every parameter cotangent of every layer, the base's μ̄ / σ̄ / L̄."""
    import torch

    xd = B.from_numpy(x) if layout == "dense" else _strided(B, x, 1, x.shape[0] + 3)
    lbd = torch.from_numpy(lb.astype(f32)).cuda()
    if bd is not None:
        xbar, flow_g, base_g = B.logpdf_vjp(B.transformed(bd, dev_t), xd, lbd)
        grads = flow_g[::-1]
    else:
        yd = None if ybar is None else (B.from_numpy(ybar) if layout == "dense" else _strided(B, ybar, 3, x.shape[0] + 5))
        xbar, grads = B.chain_vjp(dev_t, xd, yd, lbd)
    kw = kw or {}
    o64 = V.chain_vjp(ora, flags, x.astype(np.float64), ybar, lb, **kw)
    o32 = V.chain_vjp(ora, flags, x, None if ybar is None else ybar.astype(f32), lb.astype(f32), dtype=f32, **kw)

    def chk(d, a64, a32, what):
        if np.size(a64) == 1 and what[1] == "b":
            # planar b̄, one column sum: test_chain_vjp.check_chain's absolute rule with a 1e-3 floor (the cotangent it
            # sums carries the ~2e-4 of the note above VJP_FLOOR; in the 23-layer chain b̄ ≈ 59 comes out 3.6e-4 off)
            b64, b32 = float(np.ravel(a64)[0]), float(np.ravel(a32)[0])
            tol = max(1e-3 * max(abs(b64), np.sqrt(x.shape[1])), 4.0 * abs(b32 - b64))
            got = float(B.to_numpy(d).ravel()[0])
            assert abs(got - b64) <= tol, (what, got, b64, b32, tol)
            return
        gate(B.to_numpy(d), np.reshape(a64, d.shape), np.reshape(a32, d.shape), what, VJP_FLOOR, 4.0)

    chk(xbar, o64[0], o32[0], "x̄")
    assert len(grads) == len(ora)
    for l, (gd, g64, g32) in enumerate(zip(grads, o64[1], o32[1])):
        assert set(gd) == set(g64), (l, set(gd), set(g64))
        for k in gd:
            chk(gd[k], g64[k], g32[k], (l, k))
    if bd is not None:
        assert set(base_g) == set(o64[2])
        for k in base_g:
            chk(base_g[k], o64[2][k], o32[2][k], k)
        if "L" in base_g:
            assert np.all(np.triu(base_g["L"].cpu().numpy(), 1) == 0.0)


# the affine coupling's VJP kernel stages 2·D rows in shared memory: D = 1024 is outside its envelope
VJP_CHAINS = [name for name in CHAINS if CHAINS[name][0] < 1024]


@pytest.mark.parametrize("mode", ["ybar", "no-ybar", "strided"])
@pytest.mark.parametrize("name", VJP_CHAINS)
def test_chain_vjp(B, name, mode):
    D, dev, ora, flags = build(B, name)
    rng = np.random.default_rng(D + 17 + len(mode))
    N = 613
    x = inputs(rng, D, N)
    ybar = None if mode == "no-ybar" else rng.standard_normal((D, N)).astype(f32)
    check_vjp(B, B.Composed(*dev), ora, flags, x, ybar, rng.standard_normal(N), layout="dense" if mode != "strided" else mode)


@pytest.mark.parametrize("name,base", [(n, b) for n, b in BASES if n in VJP_CHAINS])
def test_logpdf_vjp(B, name, base):
    D, dev, ora, flags = build(B, name)
    rng = np.random.default_rng(D + 23 + len(base))
    N = 777
    x = inputs(rng, D, N)
    bd, kw = base_of(B, rng, D, base)
    check_vjp(B, B.inverse(B.Composed(*dev)), ora, flags, x, None, rng.standard_normal(N), kw, bd)


def test_flow_training_gradients(B):
    """autograd.Flow over the D = 64 chain of every kind with a full-covariance base: every .grad against the reference."""
    D, dev, ora, flags = build(B, "every64", seed=1)
    rng = np.random.default_rng(99)
    N = 1024
    bd, kw = base_of(B, rng, D, "tril")
    F = B.autograd.Flow(B.inverse(B.Composed(*dev)), base=bd)  # logpdf pulls the data back through the chain itself
    x = inputs(rng, D, N)
    F.nll(B.from_numpy(x)).backward()
    lb = -np.ones(N)  # the cotangent of -Σ logpdf
    o64 = V.chain_vjp(ora, flags, x.astype(np.float64), None, lb, **kw)
    o32 = V.chain_vjp(ora, flags, x, None, lb.astype(f32), dtype=f32, **kw)
    got = {p.data_ptr(): p.grad for p in F.params}
    assert all(g is not None for g in got.values())
    gate(got[bd.mu.data_ptr()].cpu().numpy(), o64[2]["μ"], o32[2]["μ"], "μ")
    gate(got[bd._tril.data_ptr()].t().cpu().numpy(), o64[2]["L"], o32[2]["L"], "L")
    checked = 2
    for l, d in enumerate(dev):
        # the trainable tensors of a leaf come in the order of the reference's cotangent dict; matrices are stored
        # column-major (transposed)
        for name, t in zip(o64[1][l], B.autograd._trainable_tensors(d)):
            g64, g32 = o64[1][l][name], o32[1][l][name]
            g = got[t.data_ptr()]
            g = (g.t() if g.dim() == 2 else g).cpu().numpy()
            checked += 1
            if np.size(g64) == 1 and name == "b":  # planar b̄: test_chain_vjp.check_chain's absolute rule
                b64, b32 = float(np.ravel(g64)[0]), float(np.ravel(g32)[0])
                assert abs(float(g.ravel()[0]) - b64) <= max(5e-5 * max(abs(b64), np.sqrt(N)), 2.0 * abs(b32 - b64)), l
                continue
            gate(g.reshape(np.shape(g64)), g64, g32, (l, name))
    assert checked == len(F.params)


# ---- batch-sum status codes ----------------------------------------------------------------------------------------------
def test_batch_sum_over_folded_batchnorm(B):
    """A batch sum over [BN, Coupling, BN] with the workspace b2b_chain_workspace_bytes reports (which folds BatchNorm into
    the coupling launch) is accepted, raw and through logabsdetjac(Columnwise(...)), and matches the float64 Σ."""
    import torch

    from bijectors_jl_b200.interface import _desc_array

    rng = np.random.default_rng(5)
    D, N = 64, 3001
    pairs = [_layer(B, rng, D, k, o) for k, o in (("bn", {}), ("cpl", dict(n1=32, n2=32)), ("bn", {}))]
    dev, ora = [p for p, _ in pairs], [o for _, o in pairs]
    x = inputs(rng, D, N)
    s64 = float(V.chain_logjac(ora, [False] * 3, x.astype(np.float64))[1].sum())
    descs = B.Composed(*dev)._descs(False, D)
    arr, L = _desc_array(descs), len(descs)
    xd = B.from_numpy(x)
    out = torch.empty((), dtype=torch.float64, device="cuda")
    lj = torch.empty(N, device="cuda")
    assert _run(B, arr, L, D, N, xd.data_ptr(), D, None, D, lj.data_ptr(), 0, out.data_ptr(), 1) == 0
    assert abs(float(out) - s64) <= 1e-5 * abs(s64)
    assert abs(float(out) - float(lj.double().sum())) <= 1e-9 * abs(float(out))
    total = B.logabsdetjac(B.Columnwise(B.Composed(*dev)), xd)
    assert float(total) == float(out)


@pytest.mark.parametrize("last", ["spl", "mlp", "scale"])
def test_batch_sum_after_own_launch_is_refused(B, last):
    """A chain ending in a spline, MLP or Scale launch has no fused launch to reduce the batch sum in."""
    import torch

    from bijectors_jl_b200.interface import _desc_array

    rng = np.random.default_rng(3)
    D, N = 32, 100
    o = dict(scale={}, spl=dict(n1=16, n2=16), mlp=dict(n1=16, n2=16, H=8))[last]
    dev = [_layer(B, rng, D, "planar", {})[0], _layer(B, rng, D, last, o)[0]]
    descs = B.Composed(*dev)._descs(False, D)
    arr = _desc_array(descs)
    x = B.from_numpy(inputs(rng, D, N))
    lj = torch.full((N,), 3.5, device="cuda")
    out = torch.full((), 3.5, dtype=torch.float64, device="cuda")
    rc = _run(B, arr, 2, D, N, x.data_ptr(), D, None, D, lj.data_ptr(), 0, out.data_ptr(), 1)
    assert rc == B._lib.B2B_EUNSUPPORTED
    assert float(out) == 3.5 and (lj == 3.5).all()
