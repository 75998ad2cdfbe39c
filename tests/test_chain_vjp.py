"""GPU tests of b2b_chain_vjp_f32 (reverse mode through any chain), chain_vjp / logpdf_vjp and autograd.Flow against the
float64 restatements of tests/chain_vjp_oracle.py, within the parity gate of test_gpu_parity (1e-5 norm-wise, or twice the
oracle's own float32 error on the same input)."""
import ctypes
import zlib

import numpy as np
import pytest

import chain_vjp_oracle as V
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5
EW = O.EW
INF = float("inf")


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


# (code, a, b, input range of the forward direction)
LAWS = {
    "identity": (EW.IDENTITY, 0.0, 0.0), "exp": (EW.EXP, 0.0, 0.0), "log": (EW.LOG, 0.0, 0.0), "shift": (EW.SHIFT, 0.7, 0.0),
    "scale": (EW.SCALE, -1.7, 0.0), "leaky_relu": (EW.LEAKY_RELU, 0.1, 0.0), "logit": (EW.LOGIT, -1.0, 3.0),
    "truncated": (EW.TRUNCATED, -1.0, 3.0), "truncated_lo": (EW.TRUNCATED, -1.0, INF), "truncated_hi": (EW.TRUNCATED, -INF, 3.0),
    "truncated_inf": (EW.TRUNCATED, -INF, INF),
}


def law_bijector(B, name):
    code, a, b = LAWS[name]
    return {EW.IDENTITY: lambda: B.Shift(0.0), EW.EXP: lambda: B.elementwise("exp"), EW.LOG: lambda: B.elementwise("log"),
            EW.SHIFT: lambda: B.Shift(a), EW.SCALE: lambda: B.Scale(a), EW.LEAKY_RELU: lambda: B.LeakyReLU(a),
            EW.LOGIT: lambda: B.Logit(a, b), EW.TRUNCATED: lambda: B.TruncatedBijector(a, b)}[code]()


def law_op(name):
    code, a, b = LAWS[name]
    if name == "identity":
        return (EW.SHIFT, f32(0.0))
    return (code, f32(a), f32(b)) if code in (EW.LOGIT, EW.TRUNCATED) else (code, f32(a))


def law_inputs(name, inverse, rng, shape):
    """Inputs in the domain of the law (or of its inverse); Truncated forward inputs also lie outside the box."""
    code = LAWS[name][0]
    if not inverse:
        if code == EW.LOG:
            return rng.uniform(0.2, 3.0, shape)
        if code == EW.LOGIT:
            return rng.uniform(-0.9, 2.9, shape)
        if code == EW.TRUNCATED:
            x = rng.uniform(-0.9, 2.9, shape)
            x[:, ::7] = rng.uniform(-3.0, 5.0, (shape[0], x[:, ::7].shape[1]))
            return x
        return rng.standard_normal(shape)
    if code == EW.EXP:
        return rng.uniform(0.2, 3.0, shape)
    return rng.standard_normal(shape)


def stacked_case(B, names, D):
    """Stacked of the given laws over (nearly) equal row ranges: (device layer, oracle layer, ranges)."""
    k = len(names)
    cuts = [round(i * D / k) for i in range(k + 1)]
    ranges = [(cuts[i] + 1, cuts[i + 1]) for i in range(k) if cuts[i + 1] > cuts[i]]
    names = [n for i, n in enumerate(names) if cuts[i + 1] > cuts[i]]
    return (B.Stacked([law_bijector(B, n) for n in names], ranges),
            O.Layer("stacked", dict(ops=[law_op(n) for n in names], ranges=ranges)))


def check_chain(B, dev_t, olayers, flags, x, ybar, ljbar, mu=None, sigma=None, base=None, terminal=False):
    """Device chain_vjp / logpdf_vjp against the oracle (x̄, every layer's parameter cotangents and the base's μ̄ / σ̄)."""
    import torch

    xd = B.from_numpy(x.astype(f32))
    lb = torch.from_numpy(ljbar.astype(f32)).cuda()
    if terminal:
        ybd, flow_g, base_g = B.logpdf_vjp(B.transformed(base, dev_t), xd, lb)
        dev_grads = flow_g[::-1]  # oracle order: application order of inverse(flow)
    else:
        ybd, dev_grads = B.chain_vjp(dev_t, xd, None if ybar is None else B.from_numpy(ybar.astype(f32)), lb)
    o64 = V.chain_vjp(olayers, flags, x, ybar, ljbar, mu, sigma, terminal)
    o32 = V.chain_vjp(olayers, flags, x.astype(f32), ybar, ljbar, mu, sigma, terminal, dtype=np.float32)

    def chk(dev, a64, a32, what):
        if np.size(a64) == 1 and what[1] == "b":
            # planar b̄ is one column sum: absolute error against max(|b̄|, √N) as in the planar VJP tests, or twice the
            # float32 oracle's own error
            b64, b32 = float(np.ravel(a64)[0]), float(np.ravel(a32)[0])
            tol = max(5e-5 * max(abs(b64), np.sqrt(x.shape[1])), 2.0 * abs(b32 - b64))
            assert abs(float(B.to_numpy(dev).ravel()[0]) - b64) <= tol, what
            return
        tol = max(RTOL, 2.0 * rel(a32, a64))
        e = rel(B.to_numpy(dev), a64)
        assert e <= tol, (what, e, tol)

    chk(ybd, o64[0], o32[0], "x̄")
    assert len(dev_grads) == len(olayers)
    for l, (gd, g64, g32) in enumerate(zip(dev_grads, o64[1], o32[1])):
        assert set(gd) == set(g64), (l, set(gd), set(g64))
        for k in gd:
            chk(gd[k], np.reshape(g64[k], gd[k].shape), np.reshape(g32[k], gd[k].shape), (l, k))
    if terminal:
        assert set(base_g) == set(o64[2])
        for k in base_g:
            chk(base_g[k], o64[2][k], o32[2][k], k)
    return ybd, dev_grads


# ---- 1. the elementwise-run kernel --------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,N", [(3, 7), (10, 333), (32, 1000), (128, 515), (200, 129), (257, 65), (1024, 33)])
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("law", list(LAWS))
def test_stacked_law_vjp(B, law, inverse, D, N):
    rng = np.random.default_rng(zlib.crc32(f"{law}-{inverse}-{D}".encode()))
    lay, olay = stacked_case(B, [law], D)
    x = law_inputs(law, inverse, rng, (D, N))
    ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal(N)
    check_chain(B, B.inverse(lay) if inverse else lay, [olay], [inverse], x, ybar, ljbar)


@pytest.mark.parametrize("given", ["none", "mu", "sigma", "both"])
@pytest.mark.parametrize("D,N", [(10, 777), (128, 1500)])
def test_permute_between_stacked_and_mvnormal(B, given, D, N):
    rng = np.random.default_rng(D + len(given))
    s1, o1 = stacked_case(B, ["logit", "shift"], D)
    perm = (rng.permutation(D) + 1).tolist()
    s2, o2 = stacked_case(B, ["scale", "leaky_relu"], D)
    flow = B.inverse(B.Composed(s1, B.Permute(perm), s2))  # logpdf evaluates inverse(inverse(...)) = s1 -> perm -> s2
    olayers = [o1, O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))), o2]
    mu = (rng.standard_normal(D) * 0.3).astype(f32) if given in ("mu", "both") else None
    sigma = rng.uniform(0.5, 1.5, D).astype(f32) if given in ("sigma", "both") else None
    base = B.MvNormal(D, mu=mu, sigma=sigma)
    x = np.concatenate([rng.uniform(-0.9, 2.9, (D // 2, N)), rng.standard_normal((D - D // 2, N))])
    check_chain(B, flow, olayers, [False, False, False], x, None, rng.standard_normal(N), mu, sigma, base, terminal=True)


# ---- 2. the reference's documented flows ---------------------------------------------------------------------------------
def planar_pair(B, D, rng, scale=1.0):
    w, u = (rng.standard_normal(D) * scale).astype(f32), (rng.standard_normal(D) * scale).astype(f32)
    b = rng.standard_normal(1).astype(f32)
    return B.PlanarLayer(w, u, b), O.Layer("planar", dict(w=w, u=u, b=b))


def radial_pair(B, D, rng, z0_scale=1.0):
    a, be = rng.standard_normal(1).astype(f32), rng.standard_normal(1).astype(f32)
    z0 = (rng.standard_normal(D) * z0_scale).astype(f32)
    return B.RadialLayer(a, be, z0), O.Layer("radial", dict(alpha_raw=a, beta=be, z0=z0))


def test_bounded_flow_logpdf_gradient(B):
    # inverse(Stacked([elementwise(log), Logit(0, 1)])) ∘ PlanarLayer(2), docs/src/flows.md:25-36
    rng = np.random.default_rng(5)
    D, N = 2, 4001
    pl, opl = planar_pair(B, D, rng)
    st = B.Stacked([B.elementwise("log"), B.Logit(0.0, 1.0)], [(1, 1), (2, 2)])
    ost = O.Layer("stacked", dict(ops=[(EW.LOG, f32(0)), (EW.LOGIT, f32(0.0), f32(1.0))], ranges=[(1, 1), (2, 2)]))
    flow = B.ComposedFunction(B.inverse(st), pl)
    y = np.stack([rng.uniform(0.2, 3.0, N), rng.uniform(0.05, 0.95, N)])
    # logpdf applies inverse(flow) = inverse(planar) ∘ Stacked
    check_chain(B, flow, [ost, opl], [False, True], y, None, rng.standard_normal(N), base=B.MvNormal(D), terminal=True)


def test_planar_planar_radial_flow(B):
    # PlanarLayer(10) ∘ PlanarLayer(10) ∘ RadialLayer(10), docs/src/flows.md:115
    rng = np.random.default_rng(6)
    D, N = 10, 3001
    r, orr = radial_pair(B, D, rng)
    p1, op1 = planar_pair(B, D, rng, 0.3)
    p2, op2 = planar_pair(B, D, rng, 0.3)
    flow = B.compose(p2, p1, r)
    x = rng.standard_normal((D, N))
    check_chain(B, flow, [orr, op1, op2], [False] * 3, x, rng.standard_normal((D, N)), rng.standard_normal(N))
    check_chain(B, flow, [op2, op1, orr], [True] * 3, x, None, rng.standard_normal(N), base=B.MvNormal(D), terminal=True)


# ---- 3. a D = 64 chain of every kind -------------------------------------------------------------------------------------
def every_kind(B, rng, D=64):
    laws = ["identity", "exp", "log", "shift", "scale", "leaky_relu", "logit", "truncated"]
    st, ost = stacked_case(B, laws, D)
    perm = (rng.permutation(D) + 1).tolist()
    K = 8
    spl = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                    rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    W, H, Dv = spl.knots()
    n1 = D // 2
    # conditioner weights small enough that every layer's values stay O(1-10): e^s scales rows by at most a few
    c1W = (rng.standard_normal((2 * n1, D - n1)) * 0.01).astype(f32)
    c1c = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    idx1, idx2 = list(range(1, n1 + 1)), list(range(n1 + 1, D + 1))
    cp1 = B.Coupling(B.AffineConditioner(c1W, c1c), B.PartitionMask(D, idx1, idx2))
    sel = sorted(rng.choice(np.arange(1, D + 1), 20, replace=False).tolist())
    rest = [i for i in range(1, D + 1) if i not in set(sel)]
    c2W = (rng.standard_normal((40, len(rest))) * 0.01).astype(f32)
    c2c = (rng.standard_normal(40) * 0.1).astype(f32)
    cp2 = B.Coupling(B.AffineConditioner(c2W, c2c), B.PartitionMask(D, sel, rest))
    bnp = [(rng.standard_normal(D) * 0.1).astype(f32) for _ in range(3)] + [rng.uniform(0.5, 1.5, D).astype(f32)]
    bn = B.InvertibleBatchNorm(b=bnp[0], logs=bnp[1], m=bnp[2], v=bnp[3])
    pls = [planar_pair(B, D, rng, 0.05) for _ in range(10)]
    pinv = [False, False, True, True, True, False, False, False, True, False]
    rads = [radial_pair(B, D, rng, 0.1) for _ in range(3)]
    rinv = [False, True, False]
    dev = [st, B.Permute(perm), spl, cp1, bn, cp2] + [B.inverse(p) if i else p for (p, _), i in zip(pls, pinv)] + \
          [B.inverse(r) if i else r for (r, _), i in zip(rads, rinv)]
    ol = [ost, O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))),
          O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv)),
          O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=c1W, c=c1c)),
          O.Layer("batchnorm", dict(bn=O.BatchNormParams(*bnp, f32(1e-5), f32(0.1)))),
          O.Layer("coupling_affine", dict(idx1=np.asarray(sel), idx2=np.asarray(rest), W=c2W, c=c2c))] + \
         [o for _, o in pls] + [o for _, o in rads]
    flags = [False] * 6 + pinv + rinv
    return dev, ol, flags


def every_kind_inputs(rng, D, N):
    x = rng.standard_normal((D, N)) * 0.5
    x[8:24] = rng.uniform(0.2, 1.5, (16, N))  # exp / log rows of the Stacked block (the first layer; D/8 rows per law)
    x[48:56] = rng.uniform(-0.9, 2.9, (8, N))
    x[56:] = rng.uniform(-0.9, 2.9, (8, N))
    return x


def test_every_kind_chain(B):
    rng = np.random.default_rng(64)
    D, N = 64, 1537
    dev, ol, flags = every_kind(B, rng, D)
    x = every_kind_inputs(rng, D, N)
    check_chain(B, B.Composed(*dev), ol, flags, x, rng.standard_normal((D, N)), rng.standard_normal(N))


def test_every_kind_chain_logpdf(B):
    rng = np.random.default_rng(65)
    D, N = 64, 1025
    dev, ol, flags = every_kind(B, rng, D)
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.4, D).astype(f32)
    # logpdf(transformed(base, inverse(flow)), y) runs the chain `flow` itself, then the MvNormal
    x = every_kind_inputs(rng, D, N)
    flow = B.inverse(B.Composed(*dev))
    check_chain(B, flow, ol, flags, x, None, rng.standard_normal(N), mu, sigma, B.MvNormal(D, mu=mu, sigma=sigma), terminal=True)


def test_realnvp_shape_small_n(B):
    rng = np.random.default_rng(55)
    D, N = 256, 300
    n1 = 128
    dev, ol = [], []
    for l in range(2):
        idx1 = list(range(1, n1 + 1)) if l % 2 == 0 else list(range(n1 + 1, D + 1))
        idx2 = [i for i in range(1, D + 1) if i not in set(idx1)]
        W = (rng.standard_normal((2 * n1, n1)) * 0.02).astype(f32)
        c = (rng.standard_normal(2 * n1) * 0.05).astype(f32)
        dev.append(B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2)))
        ol.append(O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c)))
        bnp = [(rng.standard_normal(D) * 0.1).astype(f32) for _ in range(3)] + [rng.uniform(0.5, 1.5, D).astype(f32)]
        dev.append(B.InvertibleBatchNorm(b=bnp[0], logs=bnp[1], m=bnp[2], v=bnp[3]))
        ol.append(O.Layer("batchnorm", dict(bn=O.BatchNormParams(*bnp, f32(1e-5), f32(0.1)))))
    y = rng.standard_normal((D, N))
    check_chain(B, B.Composed(*dev), ol[::-1], [True] * 4, y, None, rng.standard_normal(N), base=B.MvNormal(D), terminal=True)


# ---- 4. single-segment chains are the per-kind entry points ------------------------------------------------------------
def test_single_segments_bit_identical(B):
    import torch

    rng = np.random.default_rng(9)
    D, N = 64, 2000
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    yb = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lb = torch.randn(N, device="cuda")
    pl = B.inverse(B.Composed(*[planar_pair(B, D, rng, 0.2)[0] for _ in range(5)]))
    xa, ga = B.chain_vjp(pl, x, yb, lb)
    xb_, gb = B.planar_chain_vjp(pl, x, yb, lb)
    assert torch.equal(xa, xb_) and all(torch.equal(a[k], b[k]) for a, b in zip(ga, gb) for k in a)
    rd = B.Composed(radial_pair(B, D, rng)[0], B.inverse(radial_pair(B, D, rng)[0]))
    xa, ga = B.chain_vjp(rd, x, yb, lb)
    xb_, gb = B.radial_chain_vjp(rd, x, yb, lb)
    assert torch.equal(xa, xb_) and all(torch.equal(a[k], b[k]) for a, b in zip(ga, gb) for k in a)
    spl = B.RationalQuadraticSpline(rng.standard_normal((D, 8)).astype(f32), rng.standard_normal((D, 8)).astype(f32),
                                    rng.standard_normal((D, 7)).astype(f32), 3.0)
    cp = B.Coupling(B.AffineConditioner((rng.standard_normal((64, 32)) * 0.1).astype(f32), np.zeros(64, f32)),
                    B.PartitionMask(D, list(range(1, 33))))
    bn = B.InvertibleBatchNorm(b=np.zeros(D, f32), logs=(rng.standard_normal(D) * 0.1).astype(f32), m=np.zeros(D, f32), v=np.ones(D, f32))
    for lay, fn in ((spl, B.rqs_vjp), (B.inverse(cp), B.coupling_vjp), (bn, B.batchnorm_vjp)):
        xa, ga = B.chain_vjp(lay, x, yb, lb)
        xb_, gb = fn(lay, x, yb, lb)
        assert torch.equal(xa, xb_) and all(torch.equal(ga[0][k], gb[k]) for k in gb)


# ---- 5. edge cases and status codes --------------------------------------------------------------------------------------
def _raw(B, descs, x, ybar, ljbar, xbar, bars, D, N, ldx, ldyb, ldxb, ws_bytes=None):
    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200.interface import _desc_array, _stream

    L_ = _lib.lib()
    arr = _desc_array(descs)
    need = L_.b2b_chain_vjp_workspace_bytes(arr, len(descs), D, N)
    import torch

    ws = torch.empty((max(need, 1),), dtype=torch.uint8, device="cuda")
    return L_.b2b_chain_vjp_f32(arr, len(descs), x, ybar, ljbar, xbar, bars, D, N, ldx, ldyb, ldxb, ws.data_ptr(),
                                need if ws_bytes is None else ws_bytes, _stream())


def test_edge_cases_and_status_codes(B):
    import torch

    from bijectors_jl_b200 import _lib

    rng = np.random.default_rng(12)
    D = 40
    st, _ = stacked_case(B, ["exp", "scale"], D)
    pl = planar_pair(B, D, rng, 0.2)[0]
    chain = B.Composed(st, pl, B.Permute((rng.permutation(D) + 1).tolist()))
    descs = chain._descs(False, D)
    for N in (0, 1, 5):
        x = torch.randn(N, D + 3, device="cuda").t()[:D]  # padded ld
        yb = torch.randn(N, D + 1, device="cuda").t()[:D]
        xb = torch.empty(N, D + 5, device="cuda").t()[:D]
        wbar = torch.full((D,), 7.0, device="cuda")
        bars = (ctypes.c_void_p * (4 * len(descs)))()
        bars[4 * 1 + 0] = wbar.data_ptr()  # only w̄ of the planar layer
        rc = _raw(B, descs, x.data_ptr() if N else None, yb.data_ptr() if N else None, None, xb.data_ptr() if N else None,
                  ctypes.cast(bars, ctypes.c_void_p), D, N, D + 3, D + 1, D + 5)
        assert rc == 0, rc
        torch.cuda.synchronize()
        if N == 0:
            assert torch.count_nonzero(wbar) == 0
        else:
            ref, g = B.chain_vjp(chain, B.from_numpy(B.to_numpy(x)), B.from_numpy(B.to_numpy(yb)))
            assert torch.equal(xb, ref) and torch.equal(wbar, g[1]["w"])
    N = 100
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    xb = B.colmajor_empty(D, N)
    # NULL ybar / ljbar / param_bars
    assert _raw(B, descs, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D) == 0
    torch.cuda.synchronize()
    assert torch.count_nonzero(xb) == 0
    # overlapping x̄
    assert _raw(B, descs, x.data_ptr(), None, None, x.data_ptr(), None, D, N, D, D, D) == _lib.B2B_EINVAL
    # short workspace
    assert _raw(B, descs, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, ws_bytes=64) == _lib.B2B_EWORKSPACE
    # a cotangent of a Stacked layer, D beyond the planar limit, training-mode BatchNorm
    bars = (ctypes.c_void_p * (4 * len(descs)))()
    bars[0] = xb.data_ptr()
    assert _raw(B, descs, x.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(bars, ctypes.c_void_p), D, N, D, D, D) == _lib.B2B_EUNSUPPORTED
    Dw = 130
    big = planar_pair(B, Dw, rng)[0]
    xw = B.from_numpy(rng.standard_normal((Dw, 8)).astype(f32))
    with pytest.raises(B.B2BError) as ei:
        B.chain_vjp(big, xw)
    assert ei.value.status == _lib.B2B_EUNSUPPORTED
    with pytest.raises(B.B2BError) as ei:
        B.autograd.Flow(B.InvertibleBatchNorm(D, training=True))
    assert ei.value.status == _lib.B2B_EUNSUPPORTED


def test_deterministic_and_graph_capture(B):
    import torch

    rng = np.random.default_rng(13)
    D, N = 64, 5000
    dev, _, _ = every_kind(B, rng, D)
    flow = B.Composed(*dev)
    x = B.from_numpy(every_kind_inputs(rng, D, N).astype(f32))
    yb = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lb = torch.randn(N, device="cuda")
    a = B.chain_vjp(flow, x, yb, lb)
    b = B.chain_vjp(flow, x, yb, lb)
    assert torch.equal(a[0], b[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], b[1]) for k in p)
    out = {}
    g = B.GraphedCalls(lambda: out.__setitem__("r", B.chain_vjp(flow, x, yb, lb)))
    c = out["r"]
    c[0].fill_(float("nan"))
    g()
    torch.cuda.synchronize()
    assert torch.equal(a[0], c[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], c[1]) for k in p)


# ---- 6. autograd.Flow ----------------------------------------------------------------------------------------------------
def test_flow_gradients_match_oracle(B):
    import torch

    rng = np.random.default_rng(21)
    D, N = 64, 700
    dev, ol, flags = every_kind(B, rng, D)
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.4, D).astype(f32)
    base = B.MvNormal(D, mu=mu, sigma=sigma)
    model = B.autograd.Flow(B.inverse(B.Composed(*dev)), base)
    x = every_kind_inputs(rng, D, N)
    lp = model.logpdf(B.from_numpy(x.astype(f32)))
    lp.sum().backward()
    o = V.chain_vjp(ol, flags, x, None, np.ones(N), mu, sigma, terminal=True)
    o32 = V.chain_vjp(ol, flags, x.astype(f32), None, np.ones(N), mu, sigma, terminal=True, dtype=np.float32)
    got = {p.data_ptr(): p.grad for p in model.params}
    leaf_tensors = B.autograd._trainable_tensors
    for l, d in enumerate(dev):
        kind_names = {"PlanarLayer": ("w", "u", "b"), "RadialLayer": ("α_", "β", "z_0"),
                      "RationalQuadraticSpline": ("widths", "heights", "derivatives"), "Coupling": ("W", "c"),
                      "InvertibleBatchNorm": ("b", "logs")}
        lay = d.orig if isinstance(d, B.Inverse) else d
        for name, t in zip(kind_names.get(type(lay).__name__, ()), leaf_tensors(d)):
            g64, g32 = o[1][l][name], o32[1][l][name]
            dev_g = got[t.data_ptr()]
            if name in ("widths", "heights", "derivatives", "W"):
                dev_g = dev_g.t()
            if name == "b" and np.size(g64) == 1:  # planar b̄: as in check_chain
                b64, b32 = float(np.ravel(g64)[0]), float(np.ravel(g32)[0])
                assert abs(float(dev_g.item()) - b64) <= max(5e-5 * max(abs(b64), np.sqrt(N)), 2.0 * abs(b32 - b64)), l
                continue
            tol = max(RTOL, 2 * rel(g32, g64))
            assert rel(B.to_numpy(dev_g).reshape(np.shape(g64)), g64) <= tol, (l, name)
    for name, t in (("μ", base.mu), ("σ", base.sigma)):
        tol = max(RTOL, 2 * rel(o32[2][name], o[2][name]))
        assert rel(B.to_numpy(got[t.data_ptr()]), o[2][name]) <= tol, name


def test_bounded_flow_trains_by_nll(B):
    import torch

    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    D, N = 2, 4096
    pl = B.PlanarLayer((rng.standard_normal(D) * 0.5).astype(f32), (rng.standard_normal(D) * 0.5).astype(f32), np.zeros(1, f32))
    st = B.Stacked([B.elementwise("log"), B.Logit(0.0, 1.0)], [(1, 1), (2, 2)])
    model = B.autograd.Flow(B.ComposedFunction(B.inverse(st), pl))
    # data: a log-normal first coordinate and a Beta-like second one
    y = torch.stack([torch.exp(0.5 * torch.randn(N) + 0.3), torch.sigmoid(0.7 * torch.randn(N) - 0.4)]).cuda()
    y = y.t().contiguous().t()
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    losses = []
    for it in range(300):
        opt.zero_grad()
        loss = model.nll(y) / N
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert np.isfinite(losses).all() and np.mean(losses[-20:]) < np.mean(losses[:20]) - 0.05, (losses[:3], losses[-3:])


# ---- 7. the headline shape -----------------------------------------------------------------------------------------------
def test_headline_logpdf_gradient(B):
    import torch

    rng = np.random.default_rng(1)
    D, N, L = 128, 1 << 20, 8
    pairs = [planar_pair(B, D, rng, 1 / np.sqrt(D)) for _ in range(L)]
    flow = B.Composed(*[p for p, _ in pairs])
    y = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    ones = torch.ones(N, device="cuda")
    yb, flow_g, _ = B.logpdf_vjp(B.transformed(B.MvNormal(D), flow), y, ones)
    # today's route: planar_chain_vjp of inverse(flow) with the base density's cotangent −x computed in torch
    x, _ = B.run_chain(B.inverse(flow), y)
    xr, gr = B.planar_chain_vjp(B.inverse(flow), y, (-x).t().contiguous().t(), ones)
    assert rel(B.to_numpy(yb), B.to_numpy(xr)) <= RTOL
    for a, b in zip(flow_g, gr[::-1]):
        for k in a:
            assert rel(B.to_numpy(a[k]), B.to_numpy(b[k])) <= 1e-4, k
    # a 1024-column sample against the oracle
    ys = B.to_numpy(y[:, :1024])
    check_chain(B, flow, [o for _, o in pairs][::-1], [True] * L, ys, None, np.ones(1024), base=B.MvNormal(D), terminal=True)
