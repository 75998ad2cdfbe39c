"""GPU tests of b2b_chain_vjp_f64 (reverse mode through any Float64 chain), and of chain_vjp / logpdf_vjp / autograd.Flow on
Float64 batches, against the float64 restatements of tests/chain_vjp_oracle.py and against central differences of the
Float64 forward kernel (torch.autograd.gradcheck, the analogue of the reference's test_rrule checks).

Gate: 1e-10 norm-wise relative for x̄ and every parameter cotangent.  Column-summed scalars (planar b̄, radial ᾱ_ / β̄) are
one sum over N columns whose terms cancel: their error is held to 1e-10 · max(|ref|, 1e-2·√N), the absolute floor the
Float64 forward tests use for logjac.  Permute moves values only, so its x̄ is bit-exact."""
import ctypes
import math
import zlib

import numpy as np
import pytest

import chain_vjp_oracle as V
from oracle import oracle_np as O
from test_chain_vjp import LAWS, every_kind_inputs, law_bijector, law_inputs
from test_gpu_parity import make_case64

pytestmark = pytest.mark.gpu
f64 = np.float64
TOL = 1e-10
EW = O.EW


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def _t64():
    import torch

    return torch.float64


def _dev(B, a):
    return B.from_numpy(np.asarray(a, f64), dtype=f64)


def _vec(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, f64)).cuda()


def check_grad(dev, ref, N, what, tol=TOL):
    dev = np.asarray(dev, f64).reshape(np.shape(ref))
    if np.size(ref) == 1:  # a column sum (planar b̄, radial ᾱ_, β̄)
        r = float(np.ravel(ref)[0])
        assert abs(float(dev.ravel()[0]) - r) <= tol * max(abs(r), 1e-2 * math.sqrt(N)), (what, float(dev.ravel()[0]), r)
        return
    e = rel(dev, ref)
    assert e <= tol, (what, e)


def check_chain64(B, dev_t, olayers, flags, x, ybar, ljbar, mu=None, sigma=None, base=None, terminal=False, tol=TOL):
    """Device chain_vjp / logpdf_vjp on a Float64 batch against the float64 oracle: x̄, every layer's parameter
    cotangents and the base's μ̄ / σ̄."""
    N = x.shape[1]
    xd = _dev(B, x)
    lb = _vec(ljbar)
    if terminal:
        ybd, flow_g, base_g = B.logpdf_vjp(B.transformed(base, dev_t), xd, lb)
        dev_grads = flow_g[::-1]  # oracle order: application order of inverse(flow)
    else:
        ybd, dev_grads = B.chain_vjp(dev_t, xd, None if ybar is None else _dev(B, ybar), lb)
    assert str(ybd.dtype) == "torch.float64"
    o = V.chain_vjp(olayers, flags, x, ybar, ljbar, mu, sigma, terminal, dtype=f64)
    check_grad(B.to_numpy(ybd), o[0], N, "x̄", tol)
    assert len(dev_grads) == len(olayers)
    for l, (gd, g64) in enumerate(zip(dev_grads, o[1])):
        assert set(gd) == set(g64), (l, set(gd), set(g64))
        for k in gd:
            assert str(gd[k].dtype) == "torch.float64"
            check_grad(B.to_numpy(gd[k]), np.reshape(g64[k], gd[k].shape), N, (l, k), tol)
    if terminal:
        assert set(base_g) == set(o[2])
        for k in base_g:
            check_grad(B.to_numpy(base_g[k]), o[2][k], N, k, tol)
    return ybd, dev_grads, o


# ---- 1. every kind, both directions --------------------------------------------------------------------------------------
DS = [(3, 7), (33, 65), (128, 129), (1000, 33), (2048, 17)]


def rqs64(B, D, K, rng):
    rw, rh, rd = rng.standard_normal((D, K)), rng.standard_normal((D, K)), rng.standard_normal((D, K - 1))
    lay = B.RationalQuadraticSpline(rw, rh, rd, 3.0, dtype=_t64())
    W, H, Dv = lay.knots()
    return lay, O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv))


def rqs_raw64(B, D, K, rng, first_w=-1.0, first_h=-1.2, Bx=3.0):
    """A spline from raw three-argument knots (rational_quadratic_spline.jl:80-97): the normalised knots mapped from
    [−B, B] onto [first, B], so the first knot lies right of −B.  Inputs between −widths[end] and widths[1] (the observed
    side: heights) fall in the k = 0 bin, whose left knot is (−widths[end], −heights[end]) with the constant derivative 1."""
    _, o = rqs64(B, D, K, rng)
    W = first_w + (o.params["widths"] + Bx) * (Bx - first_w) / (2 * Bx)
    H = first_h + (o.params["heights"] + Bx) * (Bx - first_h) / (2 * Bx)
    lay = B.RationalQuadraticSpline(W, H, o.params["derivs"], dtype=_t64())
    W2, H2, D2 = lay.knots()
    assert np.all(W2[:, 0] > -Bx) and np.all(H2[:, 0] > -Bx)
    return lay, O.Layer("rqs", dict(widths=W2, heights=H2, derivs=D2))


def coupling64(B, D, idx1, idx2, rng):
    n1, n2 = len(idx1), len(idx2)
    W = rng.standard_normal((2 * n1, n2)) * 0.2 / np.sqrt(n2)
    c = rng.standard_normal(2 * n1) * 0.1
    return (B.Coupling(B.AffineConditioner(W, c, dtype=_t64()), B.PartitionMask(D, idx1, idx2)),
            O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c)))


def scattered_mask(D, rng):
    """Scattered index lists that leave about a quarter of the rows passing through."""
    perm = rng.permutation(np.arange(1, D + 1))
    n1 = max(1, D // 4)
    n2 = max(1, min(D - n1, D // 2))
    return sorted(perm[:n1].tolist()), sorted(perm[n1:n1 + n2].tolist())


def kind_case(B, kind, D, rng):
    if kind == "rqs_k5":  # a bin count that is not a power of two
        return rqs64(B, D, 5, rng)
    if kind == "rqs_raw":
        return rqs_raw64(B, D, 8, rng)
    if kind == "coupling_scattered":
        return coupling64(B, D, *scattered_mask(D, rng), rng)
    return make_case64(kind, D, rng)


KINDS = ["planar", "radial", "rqs", "rqs_k5", "rqs_raw", "coupling", "coupling_scattered", "batchnorm", "permute", "stacked", "bounded",
         "leaky_relu"]


@pytest.mark.parametrize("D,N", DS)
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_kind_vjp_f64(B, kind, inverse, D, N):
    if kind in ("coupling", "coupling_scattered", "stacked", "bounded") and D < 3:
        pytest.skip("needs D >= 3")
    rng = np.random.default_rng(zlib.crc32(f"vjp64-{kind}-{inverse}-{D}".encode()))
    lay, olay = kind_case(B, kind, D, rng)
    x = rng.standard_normal((D, N)) * (1.5 if kind.startswith("rqs") else 1.0)
    if kind == "bounded":  # inputs outside the Truncated boxes: test_stacked_law_vjp_f64
        x = rng.uniform(-0.9, 2.9, (D, N))
    if kind == "rqs_raw":  # every third column inside the k = 0 bin of its row
        S = olay.params["heights" if inverse else "widths"]
        lo, hi = -S[:, -1:], S[:, :1]
        x[:, ::3] = lo + (hi - lo) * rng.uniform(0.05, 0.95, (D, x[:, ::3].shape[1]))
        assert np.count_nonzero((x > lo) & (x <= hi)) >= D
    ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal(N)
    ybd, _, o = check_chain64(B, B.inverse(lay) if inverse else lay, [olay], [inverse], x, ybar, ljbar)
    if kind == "permute":
        assert np.array_equal(B.to_numpy(ybd).view(np.uint64), np.asarray(o[0], f64).view(np.uint64))


def stacked_law64(B, name, D):
    code, a, b = LAWS[name]
    op = (EW.SHIFT, 0.0) if name == "identity" else ((code, a, b) if code in (EW.LOGIT, EW.TRUNCATED) else (code, a))
    return (B.Stacked([law_bijector(B, name)], [(1, D)], dtype=_t64()),
            O.Layer("stacked", dict(ops=[op], ranges=[(1, D)])))


@pytest.mark.parametrize("D,N", DS)
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("law", list(LAWS))
def test_stacked_law_vjp_f64(B, law, inverse, D, N):
    rng = np.random.default_rng(zlib.crc32(f"vjp64-law-{law}-{inverse}-{D}".encode()))
    lay, olay = stacked_law64(B, law, D)
    x = law_inputs(law, inverse, rng, (D, N))
    check_chain64(B, B.inverse(lay) if inverse else lay, [olay], [inverse], x, rng.standard_normal((D, N)),
                  rng.standard_normal(N))


@pytest.mark.parametrize("given", ["none", "both"])
def test_permute_stacked_mvnormal_f64(B, given):
    rng = np.random.default_rng(77 + len(given))
    D, N = 40, 301
    l1, o1 = stacked_law64(B, "logit", D)
    perm = (rng.permutation(D) + 1).tolist()
    l2, o2 = stacked_law64(B, "scale", D)
    flow = B.inverse(B.Composed(l1, B.Permute(perm), l2))
    olayers = [o1, O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))), o2]
    mu = rng.standard_normal(D) * 0.3 if given == "both" else None
    sigma = rng.uniform(0.5, 1.5, D) if given == "both" else None
    base = B.MvNormal(D, mu=mu, sigma=sigma, dtype=_t64())
    x = rng.uniform(-0.9, 2.9, (D, N))
    check_chain64(B, flow, olayers, [False] * 3, x, None, rng.standard_normal(N), mu, sigma, base, terminal=True)


# ---- 2. whole chains -----------------------------------------------------------------------------------------------------
def planar64(B, D, rng, scale=1.0):
    w, u, b = rng.standard_normal(D) * scale, rng.standard_normal(D) * scale, rng.standard_normal(1)
    return B.PlanarLayer(w, u, b, dtype=_t64()), O.Layer("planar", dict(w=w, u=u, b=b))


def radial64(B, D, rng, z0_scale=1.0):
    a, be, z0 = rng.standard_normal(1), rng.standard_normal(1), rng.standard_normal(D) * z0_scale
    return B.RadialLayer(a, be, z0, dtype=_t64()), O.Layer("radial", dict(alpha_raw=a, beta=be, z0=z0))


def bounded_flow64(B, rng):
    """inverse(Stacked([elementwise(log), Logit(0, 1)])) ∘ PlanarLayer(2), docs/src/flows.md:25-36."""
    pl, opl = planar64(B, 2, rng, 0.5)
    st = B.Stacked([B.elementwise("log"), B.Logit(0.0, 1.0)], [(1, 1), (2, 2)], dtype=_t64())
    ost = O.Layer("stacked", dict(ops=[(EW.LOG, 0.0), (EW.LOGIT, 0.0, 1.0)], ranges=[(1, 1), (2, 2)]))
    return pl, st, B.ComposedFunction(B.inverse(st), pl), [ost, opl]


def test_bounded_flow_logpdf_gradient_f64(B):
    rng = np.random.default_rng(5)
    N = 2001
    _, _, flow, ol = bounded_flow64(B, rng)
    y = np.stack([rng.uniform(0.2, 3.0, N), rng.uniform(0.05, 0.95, N)])
    # logpdf applies inverse(flow) = inverse(planar) ∘ Stacked
    check_chain64(B, flow, ol, [False, True], y, None, rng.standard_normal(N), base=B.MvNormal(2, dtype=_t64()),
                  terminal=True)


def test_planar_planar_radial_flow_f64(B):
    # PlanarLayer(10) ∘ PlanarLayer(10) ∘ RadialLayer(10), docs/src/flows.md:115
    rng = np.random.default_rng(6)
    D, N = 10, 1501
    r, orr = radial64(B, D, rng)
    p1, op1 = planar64(B, D, rng, 0.3)
    p2, op2 = planar64(B, D, rng, 0.3)
    flow = B.compose(p2, p1, r)
    x = rng.standard_normal((D, N))
    check_chain64(B, flow, [orr, op1, op2], [False] * 3, x, rng.standard_normal((D, N)), rng.standard_normal(N))
    check_chain64(B, flow, [op2, op1, orr], [True] * 3, x, None, rng.standard_normal(N), base=B.MvNormal(D, dtype=_t64()),
                  terminal=True)


def every_kind64(B, rng, D=64):
    """The D = 64 chain of every kind of test_chain_vjp.every_kind, with Float64 parameters."""
    t = _t64()
    laws = ["identity", "exp", "log", "shift", "scale", "leaky_relu", "logit", "truncated"]
    k = len(laws)
    cuts = [round(i * D / k) for i in range(k + 1)]
    ranges = [(cuts[i] + 1, cuts[i + 1]) for i in range(k)]
    st = B.Stacked([law_bijector(B, n) for n in laws], ranges, dtype=t)
    ops = []
    for n in laws:
        code, a, b = LAWS[n]
        ops.append((EW.SHIFT, 0.0) if n == "identity" else ((code, a, b) if code in (EW.LOGIT, EW.TRUNCATED) else (code, a)))
    ost = O.Layer("stacked", dict(ops=ops, ranges=ranges))
    perm = (rng.permutation(D) + 1).tolist()
    spl, ospl = rqs64(B, D, 8, rng)
    n1 = D // 2
    c1W, c1c = rng.standard_normal((2 * n1, D - n1)) * 0.01, rng.standard_normal(2 * n1) * 0.1
    idx1, idx2 = list(range(1, n1 + 1)), list(range(n1 + 1, D + 1))
    cp1 = B.Coupling(B.AffineConditioner(c1W, c1c, dtype=t), B.PartitionMask(D, idx1, idx2))
    sel = sorted(rng.choice(np.arange(1, D + 1), 20, replace=False).tolist())
    rest = [i for i in range(1, D + 1) if i not in set(sel)]
    c2W, c2c = rng.standard_normal((40, len(rest))) * 0.01, rng.standard_normal(40) * 0.1
    cp2 = B.Coupling(B.AffineConditioner(c2W, c2c, dtype=t), B.PartitionMask(D, sel, rest))
    bnp = [rng.standard_normal(D) * 0.1 for _ in range(3)] + [rng.uniform(0.5, 1.5, D)]
    bn = B.InvertibleBatchNorm(b=bnp[0], logs=bnp[1], m=bnp[2], v=bnp[3], dtype=t)
    pls = [planar64(B, D, rng, 0.05) for _ in range(10)]
    pinv = [False, False, True, True, True, False, False, False, True, False]
    rads = [radial64(B, D, rng, 0.1) for _ in range(3)]
    rinv = [False, True, False]
    dev = [st, B.Permute(perm), spl, cp1, bn, cp2] + [B.inverse(p) if i else p for (p, _), i in zip(pls, pinv)] + \
          [B.inverse(r) if i else r for (r, _), i in zip(rads, rinv)]
    ol = [ost, O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))), ospl,
          O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=c1W, c=c1c)),
          O.Layer("batchnorm", dict(bn=O.BatchNormParams(*bnp, bn.eps, 0.1))),
          O.Layer("coupling_affine", dict(idx1=np.asarray(sel), idx2=np.asarray(rest), W=c2W, c=c2c))] + \
         [o for _, o in pls] + [o for _, o in rads]
    flags = [False] * 6 + pinv + rinv
    return dev, ol, flags


def test_every_kind_chain_f64(B):
    rng = np.random.default_rng(64)
    D, N = 64, 777
    dev, ol, flags = every_kind64(B, rng, D)
    x = every_kind_inputs(rng, D, N)
    check_chain64(B, B.Composed(*dev), ol, flags, x, rng.standard_normal((D, N)), rng.standard_normal(N))


def test_every_kind_chain_logpdf_f64(B):
    rng = np.random.default_rng(65)
    D, N = 64, 513
    dev, ol, flags = every_kind64(B, rng, D)
    mu, sigma = rng.standard_normal(D) * 0.2, rng.uniform(0.7, 1.4, D)
    x = every_kind_inputs(rng, D, N)
    flow = B.inverse(B.Composed(*dev))  # logpdf(transformed(base, inverse(flow)), y) runs `flow` itself, then the MvNormal
    check_chain64(B, flow, ol, flags, x, None, rng.standard_normal(N), mu, sigma,
                  B.MvNormal(D, mu=mu, sigma=sigma, dtype=_t64()), terminal=True)


def test_chain_of_max_length_f64(B):
    from bijectors_jl_b200 import _lib

    rng = np.random.default_rng(24)
    D, N = 24, 300
    pairs = []
    for l in range(_lib.MAX_CHAIN):
        kind = ["planar", "radial", "batchnorm", "permute", "rqs", "coupling"][l % 6]
        pairs.append(planar64(B, D, rng, 0.2) if kind == "planar" else
                     radial64(B, D, rng, 0.2) if kind == "radial" else make_case64(kind, D, rng))
    flags = [bool(rng.integers(0, 2)) for _ in pairs]
    flow = B.Composed(*[B.inverse(p) if f else p for (p, _), f in zip(pairs, flags)])
    x = rng.standard_normal((D, N))
    check_chain64(B, flow, [o for _, o in pairs], flags, x, rng.standard_normal((D, N)), rng.standard_normal(N))


# ---- 3. central differences of the Float64 forward kernel ----------------------------------------------------------------
def small_flow64(B, rng, D=4):
    t = _t64()
    raw, _ = rqs_raw64(B, D, 4, rng)  # first: the test puts inputs in its k = 0 bin
    pl, _ = planar64(B, D, rng, 0.5)
    rd, _ = radial64(B, D, rng, 0.5)
    spl, _ = rqs64(B, D, 4, rng)
    cp = B.Coupling(B.AffineConditioner(rng.standard_normal((2, D - 1)) * 0.3, rng.standard_normal(2) * 0.1, dtype=t),
                    B.PartitionMask(D, [2], [1, 3, 4]))
    bn = B.InvertibleBatchNorm(b=rng.standard_normal(D) * 0.1, logs=rng.standard_normal(D) * 0.1,
                               m=rng.standard_normal(D) * 0.1, v=rng.uniform(0.5, 1.5, D), dtype=t)
    st = B.Stacked([B.Scale(1.3), B.Shift(0.2)], [(1, 2), (3, D)], dtype=t)
    pl2, _ = planar64(B, D, rng, 0.5)
    return B.Composed(raw, pl, rd, spl, B.Permute([2, 4, 1, 3]), cp, bn, st, B.inverse(pl2))


def test_gradcheck_flow_f64(B):
    import torch

    rng = np.random.default_rng(31)
    D, N = 4, 3
    flow = small_flow64(B, rng, D)
    base = B.MvNormal(D, mu=rng.standard_normal(D) * 0.2, sigma=rng.uniform(0.7, 1.4, D), dtype=torch.float64)
    model = B.autograd.Flow(flow, base)
    ps = list(model.params)
    assert all(p.dtype == torch.float64 for p in ps) and len(ps) == 3 + 3 + 3 + 3 + 2 + 2 + 3 + 2
    x0 = rng.standard_normal((D, N))
    x0[:, 0] = -2.0  # in the k = 0 bin (−widths[end], widths[1]] = (−3, −1] of the raw-knot spline on every row
    x = _dev(B, x0).requires_grad_()
    assert torch.autograd.gradcheck(lambda x_, *p: model.forward(x_), (x, *ps), eps=1e-6, atol=1e-7, rtol=1e-5)
    y = _dev(B, rng.standard_normal((D, N))).requires_grad_()
    assert torch.autograd.gradcheck(lambda y_, *p: model.inverse(y_), (y, *ps), eps=1e-6, atol=1e-7, rtol=1e-5)
    assert torch.autograd.gradcheck(lambda y_, *p: model.logpdf(y_), (y, *ps), eps=1e-6, atol=1e-7, rtol=1e-5)


# ---- 4. the contract -----------------------------------------------------------------------------------------------------
def _raw(B, descs, x, ybar, ljbar, xbar, bars, D, N, ldx, ldyb, ldxb, ws_bytes=None):
    import torch

    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200.interface import _stream

    L_ = _lib.lib()
    arr = (_lib.LayerDesc64 * len(descs))(*descs)
    need = L_.b2b_chain_vjp_workspace_bytes_f64(arr, len(descs), D, N)
    ws = torch.empty((max(need, 1),), dtype=torch.uint8, device="cuda")
    return L_.b2b_chain_vjp_f64(arr, len(descs), x, ybar, ljbar, xbar, bars, D, N, ldx, ldyb, ldxb, ws.data_ptr(),
                                need if ws_bytes is None else ws_bytes, _stream())


def test_edge_cases_and_status_codes_f64(B):
    import torch

    from bijectors_jl_b200 import _lib

    t = torch.float64
    rng = np.random.default_rng(12)
    D = 40
    st, _ = stacked_law64(B, "scale", D)
    pl = planar64(B, D, rng, 0.2)[0]
    bn = make_case64("batchnorm", D, rng)[0]
    chain = B.Composed(st, pl, B.Permute((rng.permutation(D) + 1).tolist()), bn)
    descs = chain._descs(False, D, t)
    L_ = _lib.lib()
    for N in (0, 1, 5):
        x = torch.randn(N, D + 3, device="cuda", dtype=t).t()[:D]  # padded ld
        yb = torch.randn(N, D + 1, device="cuda", dtype=t).t()[:D]
        xb = torch.empty(N, D + 5, device="cuda", dtype=t).t()[:D]
        wbar = torch.full((D,), 7.0, device="cuda", dtype=t)
        bbar = torch.full((1,), 7.0, device="cuda", dtype=t)
        bars = (ctypes.c_void_p * (4 * len(descs)))()
        bars[4 * 1 + 0] = wbar.data_ptr()  # w̄ and b̄ of the planar layer only
        bars[4 * 1 + 2] = bbar.data_ptr()
        rc = _raw(B, descs, x.data_ptr() if N else None, yb.data_ptr() if N else None, None, xb.data_ptr() if N else None,
                  ctypes.cast(bars, ctypes.c_void_p), D, N, D + 3, D + 1, D + 5)
        assert rc == 0, rc
        assert L_.b2b_last_launch_count() == (2 if N == 0 else 3)
        torch.cuda.synchronize()
        if N == 0:
            assert torch.count_nonzero(wbar) == 0 and torch.count_nonzero(bbar) == 0
        else:
            ref, g = B.chain_vjp(chain, _dev(B, B.to_numpy(x)), _dev(B, B.to_numpy(yb)))
            assert torch.equal(xb, ref) and torch.equal(wbar, g[1]["w"]) and torch.equal(bbar, g[1]["b"])
    N = 100
    x = _dev(B, rng.standard_normal((D, N)))
    xb = B.colmajor_empty(D, N, dtype=t)
    # NULL ybar / ljbar / param_bars: x̄ = 0, one launch
    assert _raw(B, descs, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D) == 0
    assert L_.b2b_last_launch_count() == 1
    torch.cuda.synchronize()
    assert torch.count_nonzero(xb) == 0
    # NULL ybar with l̄ alone is the logjac gradient
    lb = torch.ones(N, dtype=t, device="cuda")
    assert _raw(B, descs, x.data_ptr(), None, lb.data_ptr(), xb.data_ptr(), None, D, N, D, D, D) == 0
    ref, _ = B.chain_vjp(chain, x, None, lb)
    torch.cuda.synchronize()
    assert torch.equal(xb, ref)
    # overlapping x̄ (with x, and with ȳ)
    assert _raw(B, descs, x.data_ptr(), None, None, x.data_ptr(), None, D, N, D, D, D) == _lib.B2B_EINVAL
    yb = _dev(B, rng.standard_normal((D, N)))
    assert _raw(B, descs, x.data_ptr(), yb.data_ptr(), None, yb[:, 1:].data_ptr(), None, D, N - 1, D, D, D) == _lib.B2B_EINVAL
    # short workspace
    assert _raw(B, descs, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, ws_bytes=64) == _lib.B2B_EWORKSPACE
    # a cotangent of the Stacked layer, of BatchNorm m / v, of Permute
    for slot in (4 * 0 + 0, 4 * 3 + 2, 4 * 3 + 3, 4 * 2 + 0):
        bars = (ctypes.c_void_p * (4 * len(descs)))()
        bars[slot] = xb.data_ptr()
        rc = _raw(B, descs, x.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(bars, ctypes.c_void_p), D, N, D, D, D)
        assert rc == _lib.B2B_EUNSUPPORTED, (slot, rc)


def test_d_limit_f64(B):
    import torch

    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200.interface import _stream

    t = torch.float64
    L_ = _lib.lib()
    rng = np.random.default_rng(2049)
    for D, ok in ((2048, True), (2049, False)):
        lay = B.PlanarLayer(rng.standard_normal(D) / np.sqrt(D), rng.standard_normal(D) / np.sqrt(D), rng.standard_normal(1),
                            dtype=t)
        descs = lay._descs(False, D, t)
        arr = (_lib.LayerDesc64 * 1)(*descs)
        need = L_.b2b_chain_vjp_workspace_bytes_f64(arr, 1, D, 9)
        assert (need > 0) == ok
        x = _dev(B, rng.standard_normal((D, 9)))
        xb = torch.full((9, D), float("nan"), dtype=t, device="cuda").t()
        wb = torch.full((D,), float("nan"), dtype=t, device="cuda")
        bars = (ctypes.c_void_p * 4)()
        bars[0] = wb.data_ptr()
        before = (xb.clone(), wb.clone())
        ws = torch.empty((max(need, 1 << 20),), dtype=torch.uint8, device="cuda")
        rc = L_.b2b_chain_vjp_f64(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(bars, ctypes.c_void_p), D, 9,
                                  D, D, D, ws.data_ptr(), ws.numel(), _stream())
        torch.cuda.synchronize()
        if ok:
            assert rc == 0 and L_.b2b_last_launch_count() == 3
            assert torch.isfinite(wb).all()
        else:
            assert rc == _lib.B2B_EUNSUPPORTED and L_.b2b_last_launch_count() == 0
            assert torch.equal(before[0].view(torch.int64), xb.view(torch.int64))
            assert torch.equal(before[1].view(torch.int64), wb.view(torch.int64))


def test_dtype_mix_raises(B):
    import torch

    rng = np.random.default_rng(3)
    D, N = 8, 5
    x64 = _dev(B, rng.standard_normal((D, N)))
    x32 = B.from_numpy(rng.standard_normal((D, N)).astype(np.float32))
    p32 = B.PlanarLayer(rng.standard_normal(D).astype(np.float32), rng.standard_normal(D).astype(np.float32),
                        np.zeros(1, np.float32))
    p64 = planar64(B, D, rng)[0]
    with pytest.raises(TypeError):
        B.chain_vjp(p32, x64)
    with pytest.raises(TypeError):
        B.chain_vjp(p64, x32)
    with pytest.raises(ValueError):  # a cotangent of another dtype, as for Float32 batches
        B.chain_vjp(p64, x64, B.from_numpy(rng.standard_normal((D, N)).astype(np.float32)))
    with pytest.raises(TypeError):
        B.logpdf_vjp(B.transformed(B.MvNormal(D), p64), x64)  # Float32 base under a Float64 flow
    with pytest.raises(TypeError):
        B.autograd.Flow(p64).nll(x32)
    with pytest.raises(TypeError):
        B.autograd.Flow(p32).nll(x64)
    # default cotangents take the batch's dtype
    yb, g, _ = B.logpdf_vjp(B.transformed(B.MvNormal(D, dtype=torch.float64), p64), x64)
    assert yb.dtype == torch.float64 and g[0]["w"].dtype == torch.float64


# ---- 5. determinism and CUDA-graph capture -------------------------------------------------------------------------------
def test_deterministic_and_graph_capture_f64(B):
    import torch

    rng = np.random.default_rng(13)
    D, N = 64, 3000
    dev, _, _ = every_kind64(B, rng, D)
    flow = B.Composed(*dev)
    x = _dev(B, every_kind_inputs(rng, D, N))
    yb = _dev(B, rng.standard_normal((D, N)))
    lb = torch.randn(N, device="cuda", dtype=torch.float64)
    a = B.chain_vjp(flow, x, yb, lb)
    b = B.chain_vjp(flow, x, yb, lb)
    assert torch.equal(a[0], b[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], b[1]) for k in p)
    out = {}
    g = B.GraphedCalls(lambda: out.__setitem__("r", B.chain_vjp(flow, x, yb, lb)))
    c = out["r"]
    c[0].fill_(float("nan"))
    for p in c[1]:
        for k in p:
            p[k].fill_(float("nan"))
    g()
    torch.cuda.synchronize()
    assert torch.equal(a[0], c[0]) and all(torch.equal(p[k], q[k]) for p, q in zip(a[1], c[1]) for k in p)


# ---- 6. training a Float64 Flow ------------------------------------------------------------------------------------------
def test_float64_flow_trains_by_nll(B):
    import torch

    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    N = 2048
    pl, st, flow, ol = bounded_flow64(B, rng)
    model = B.autograd.Flow(flow)
    y = torch.stack([torch.exp(0.5 * torch.randn(N, dtype=torch.float64) + 0.3),
                     torch.sigmoid(0.7 * torch.randn(N, dtype=torch.float64) - 0.4)]).cuda()
    y = y.t().contiguous().t()
    # first step: the gradients of the NLL are the oracle's
    loss = model.nll(y) / N
    loss.backward()
    o = V.chain_vjp(ol, [False, True], B.to_numpy(y), None, -np.ones(N) / N, terminal=True, dtype=f64)
    for name, t in zip(("w", "u", "b"), (pl.w, pl.u, pl.b)):
        p = next(q for q in model.params if q.data_ptr() == t.data_ptr())
        check_grad(B.to_numpy(p.grad), o[1][1][name], N, name)
    opt = torch.optim.Adam(model.parameters(), lr=2e-2)
    losses = [float(loss)]
    opt.step()
    for _ in range(60):
        opt.zero_grad()
        loss = model.nll(y) / N
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert np.isfinite(losses).all() and np.mean(losses[-5:]) < losses[0] - 0.01, (losses[:3], losses[-3:])
