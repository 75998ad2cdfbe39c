"""GPU tests of B2B_ELEMENTWISE_VEC -- Shift(a), Scale(a) and LeakyReLU(a) with a trainable vector a[D] -- against the
STACKED_EW layer it equals (code[r] = the law, the same a: bit-identical y, logjac and x̄) and against the float64
reference of tests/elementwise_vec_oracle.py (ā within the parity gate of test_chain_vjp: 1e-5 norm-wise, or twice the
reference's own float32 error)."""
import zlib

import numpy as np
import pytest

import elementwise_vec_oracle as E
import test_chain_vjp as TCV
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
LAWS = {"shift": E.SHIFT, "scale": E.SCALE, "leaky_relu": E.LEAKY_RELU}


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def seed(*k):
    return np.random.default_rng(zlib.crc32("-".join(map(str, k)).encode()))


def param(law, D, rng):
    if law == E.SHIFT:
        return rng.standard_normal(D)
    if law == E.SCALE:
        return rng.uniform(0.5, 2.0, D) * rng.choice([-1.0, 1.0], D)
    return rng.uniform(0.1, 2.0, D)


def vec(B, law, a, dtype=None):
    import torch

    cls = {E.SHIFT: B.Shift, E.SCALE: B.Scale, E.LEAKY_RELU: B.LeakyReLU}[law]
    return cls(a, dtype=dtype or torch.float32)


def stacked_eq(B, lay):
    """The STACKED_EW layer equal to the vector layer ``lay``: code[r] = its law, a = the same device tensor."""
    import torch

    class StackedEq(B.Transform):
        def __init__(self):
            self.code = torch.full((lay.a.numel(),), lay.code, dtype=torch.int32, device=lay.a.device)

        def _descs(self, inverse, D, dtype=torch.float32):
            return [B.layers._desc(B._lib.STACKED_EW, inverse, i0=self.code, p0=lay.a)]

        def _keepalive(self):
            return (self.code, lay.a)

    return StackedEq()


def launches(B):
    return B.lib().b2b_last_launch_count()


def run(B, t, x, inverse):
    y, lj = B.with_logabsdet_jacobian(B.inverse(t) if inverse else t, x)
    return B.to_numpy(y), B.to_numpy(lj), launches(B)


def rel(a, b):
    return TCV.rel(a, b)


def check_chain(B, dev_t, olayers, flags, x, ybar, ljbar, mu=None, sigma=None, base=None, terminal=False):
    """Device chain_vjp / logpdf_vjp against elementwise_vec_oracle.chain_vjp (x̄, every layer's parameter cotangents
    and the base's μ̄ / σ̄), within the gate of test_chain_vjp.check_chain."""
    import torch

    xd = B.from_numpy(x.astype(f32))
    lb = torch.from_numpy(ljbar.astype(f32)).cuda()
    if terminal:
        ybd, flow_g, base_g = B.logpdf_vjp(B.transformed(base, dev_t), xd, lb)
        dev_grads = flow_g[::-1]  # oracle order: application order of inverse(flow)
    else:
        ybd, dev_grads = B.chain_vjp(dev_t, xd, None if ybar is None else B.from_numpy(ybar.astype(f32)), lb)
    o64 = E.chain_vjp(olayers, flags, x, ybar, ljbar, mu, sigma, terminal)
    o32 = E.chain_vjp(olayers, flags, x.astype(f32), ybar, ljbar, mu, sigma, terminal, dtype=np.float32)

    def chk(dev, a64, a32, what):
        if np.size(a64) == 1 and what[1] == "b":  # planar b̄, one column sum: as in test_chain_vjp
            b64, b32 = float(np.ravel(a64)[0]), float(np.ravel(a32)[0])
            tol = max(5e-5 * max(abs(b64), np.sqrt(x.shape[1])), 2.0 * abs(b32 - b64))
            assert abs(float(B.to_numpy(dev).ravel()[0]) - b64) <= tol, what
            return
        tol = max(TCV.RTOL, 2.0 * rel(a32, a64))
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


# ---- forward ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 3, 32, 129, 257, 1024])
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("law", list(LAWS))
def test_forward_matches_stacked(B, law, inverse, D):
    rng = seed("fwd", law, inverse, D)
    N = 517
    lay = vec(B, LAWS[law], param(LAWS[law], D, rng))
    pl = B.PlanarLayer(D) if D in (32, 129) else None  # a fused run with another kind
    t, t_eq = (lay, stacked_eq(B, lay)) if pl is None else (B.Composed(pl, lay), B.Composed(pl, stacked_eq(B, lay)))
    x = rng.standard_normal((D, N))
    xd = B.from_numpy(x.astype(f32))
    y, lj, nl = run(B, t, xd, inverse)
    ye, lje, nle = run(B, t_eq, xd, inverse)
    assert np.array_equal(y, ye) and np.array_equal(lj, lje) and nl == nle
    if pl is None:
        o = E.VecLayer(LAWS[law], lay.a.cpu().numpy().astype(np.float64))
        yo, ljo = (o.inverse if inverse else o.forward)(x.astype(f32).astype(np.float64))
        assert rel(y, yo) <= 1e-5 and rel(lj, ljo) <= 1e-5 + 1e-6 * (np.linalg.norm(ljo) == 0)


@pytest.mark.parametrize("law", list(LAWS))
def test_forward_padded_and_in_place(B, law):
    import torch

    rng = seed("ld", law)
    D, N = 40, 300
    lay = vec(B, LAWS[law], param(LAWS[law], D, rng))
    x = torch.randn(N, D + 5, device="cuda").t()[:D]  # ld = D + 5
    y, lj, _ = run(B, lay, x, False)
    ye, lje, _ = run(B, stacked_eq(B, lay), x, False)
    assert np.array_equal(y, ye) and np.array_equal(lj, lje)
    xi = x.clone()
    yi, lji = B.with_logabsdet_jacobian_(lay, xi)
    assert np.array_equal(B.to_numpy(yi), ye) and np.array_equal(B.to_numpy(lji), lje)


# ---- reverse mode -------------------------------------------------------------------------------------------------------
def xbar_of(B, t, x, ybar, lb, ask):
    """x̄ (and the vector layer's grads when ``ask``) of b2b_chain_vjp_f32 on the raw descriptors."""
    from bijectors_jl_b200.interface import _chain_vjp_raw, _leaf_descs

    descs, _ = _leaf_descs(t, x.shape[0])
    want = [(l, 0) for l, d in enumerate(descs) if ask and d.kind == B._lib.ELEMENTWISE_VEC]
    xb, bars = _chain_vjp_raw(descs, x, ybar, lb, want)
    return B.to_numpy(xb), {k: B.to_numpy(v) for k, v in bars.items()}


@pytest.mark.parametrize("D,N", [(3, 7), (128, 515), (257, 65), (1024, 33)])
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("law", list(LAWS))
def test_vjp_per_law(B, law, inverse, D, N):
    import torch

    rng = seed("vjp", law, inverse, D)
    a = param(LAWS[law], D, rng)
    lay = vec(B, LAWS[law], a)
    x, ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    t = B.inverse(lay) if inverse else lay
    _, grads = check_chain(B, t, [E.VecLayer(LAWS[law], lay.a.cpu().numpy())], [inverse], x, ybar, ljbar)
    assert set(grads[0]) == {"α" if law == "leaky_relu" else "a"}
    # x̄ is the STACKED_EW equivalent's, with and without ā
    xd, yd = B.from_numpy(x.astype(f32)), B.from_numpy(ybar.astype(f32))
    lb = torch.from_numpy(ljbar.astype(f32)).cuda()
    t_eq = B.inverse(stacked_eq(B, lay)) if inverse else stacked_eq(B, lay)
    xe, _ = xbar_of(B, t_eq, xd, yd, lb, False)
    x0, _ = xbar_of(B, t, xd, yd, lb, False)
    x1, b1 = xbar_of(B, t, xd, yd, lb, True)
    assert np.array_equal(x0, xe) and np.array_equal(x1, xe)
    x2, b2 = xbar_of(B, t, xd, yd, lb, True)  # deterministic
    assert np.array_equal(x2, x1) and all(np.array_equal(b1[k], b2[k]) for k in b1)


def mixed_run(B, rng, D):
    """Permute, STACKED_EW and two vector layers in one run: (device layers, oracle layers)."""
    sc, sh = param(E.SCALE, D, rng), param(E.SHIFT, D, rng)
    perm = rng.permutation(D) + 1
    perm2 = rng.permutation(D) + 1
    st, ost = TCV.stacked_case(B, ["leaky_relu", "scale", "shift"], D)
    dev = [B.Permute(perm.tolist()), vec(B, E.SCALE, sc), st, vec(B, E.SHIFT, sh), B.Permute(perm2.tolist())]
    oracle = [O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm.tolist()))),
              E.VecLayer(E.SCALE, dev[1].a.cpu().numpy()), ost, E.VecLayer(E.SHIFT, dev[3].a.cpu().numpy()),
              O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm2.tolist())))]
    return dev, oracle


@pytest.mark.parametrize("D,N", [(5, 301), (64, 1000), (1024, 40)])
def test_vjp_mixed_run_with_terminal(B, D, N):
    rng = seed("mixed", D)
    dev, orc = mixed_run(B, rng, D)
    mu, sigma = rng.standard_normal(D), rng.uniform(0.5, 2.0, D)
    base = B.MvNormal(D, mu=mu.astype(f32), sigma=sigma.astype(f32))
    x = rng.standard_normal((D, N))
    x[:, :] = np.where(np.abs(x) < 1e-3, 0.1, x)
    ljbar = rng.standard_normal(N)
    flags = [True] * len(dev)  # logpdf runs inverse(flow): the layers last to first, inverted
    check_chain(B, B.Composed(*dev), orc[::-1], flags, x, None, ljbar,
                    mu.astype(f32).astype(np.float64), sigma.astype(f32).astype(np.float64), base=base, terminal=True)


def test_vjp_mixed_run_forward(B):
    rng = seed("mixed-fwd")
    D, N = 48, 777
    dev, orc = mixed_run(B, rng, D)
    x, ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    check_chain(B, B.Composed(*dev), orc, [False] * len(dev), x, ybar, ljbar)


@pytest.mark.parametrize("kind", ["planar", "coupling", "rqs", "tril"])
def test_vjp_around_other_segments(B, kind):
    rng = seed("around", kind)
    D, N = 32, 600
    a, b = param(E.SCALE, D, rng), param(E.SHIFT, D, rng)
    s, t = vec(B, E.SCALE, a), vec(B, E.SHIFT, b)
    os_, ot = E.VecLayer(E.SCALE, s.a.cpu().numpy()), E.VecLayer(E.SHIFT, t.a.cpu().numpy())
    if kind == "planar":
        mid, omid = TCV.planar_pair(B, D, rng)
    elif kind == "coupling":
        W = (rng.standard_normal((2 * 16, 16)) * 0.2).astype(f32)
        c = (rng.standard_normal(2 * 16) * 0.1).astype(f32)
        mask = B.PartitionMask(D, list(range(1, 17)), list(range(17, 33)))
        mid = B.Coupling(B.AffineConditioner(W, c), mask)
        omid = O.Layer("coupling_affine", dict(idx1=np.arange(1, 17), idx2=np.arange(17, 33), W=W, c=c))
    elif kind == "rqs":
        K = 8
        wd, ht, dv = rng.standard_normal((D, K)), rng.standard_normal((D, K)), rng.standard_normal((D, K - 1))
        mid = B.RationalQuadraticSpline(wd.astype(f32), ht.astype(f32), dv.astype(f32), 3.0)
        W_, H_, D_ = mid.knots()
        omid = O.Layer("rqs", dict(widths=W_, heights=H_, derivs=D_))
    x, ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    if kind == "tril":
        Lm = np.tril(rng.standard_normal((D, D)) * 0.1) + np.diag(rng.uniform(0.8, 1.5, D))
        mu = rng.standard_normal(D)
        base = B.MvNormal(D, mu=mu.astype(f32), scale_tril=Lm.astype(f32))
        td = B.transformed(base, B.Composed(s, t))
        ybd, flow_g, base_g = B.logpdf_vjp(td, B.from_numpy(x.astype(f32)),
                                           __import__("torch").from_numpy(ljbar.astype(f32)).cuda())
        o64 = E.chain_vjp([ot, os_], [True, True], x, None, ljbar, mu.astype(f32).astype(np.float64),
                          scale_tril=Lm.astype(f32).astype(np.float64))
        o32 = E.chain_vjp([ot, os_], [True, True], x.astype(f32), None, ljbar, mu.astype(f32).astype(np.float64),
                          scale_tril=Lm.astype(f32).astype(np.float64), dtype=np.float32)
        for dev, k, l in ((flow_g[1], "a", 0), (flow_g[0], "a", 1)):
            tol = max(TCV.RTOL, 2.0 * rel(o32[1][l][k], o64[1][l][k]))
            assert rel(B.to_numpy(dev[k]), o64[1][l][k]) <= tol, (l, k)
        assert rel(B.to_numpy(ybd), o64[0]) <= max(TCV.RTOL, 2.0 * rel(o32[0], o64[0]))
        return
    check_chain(B, B.Composed(s, mid, t), [os_, omid, ot], [False] * 3, x, ybar, ljbar)


def test_vjp_training_batch(B):
    """N = 2²², D = 128: the per-thread, slab and CTA sums of ā over a training-size batch."""
    import torch

    D, N = 128, 1 << 22
    rng = seed("big")
    s, t = vec(B, E.SCALE, param(E.SCALE, D, rng)), vec(B, E.SHIFT, param(E.SHIFT, D, rng))
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(N, D, device="cuda", generator=g).t()
    yb = torch.randn(N, D, device="cuda", generator=g).t()
    lb = torch.randn(N, device="cuda", generator=g)
    _, grads = B.chain_vjp(B.Composed(s, t), x, yb, lb)
    X, Y, LB = (v.double().cpu().numpy() for v in (x, yb, lb))
    a, b = s.a.double().cpu().numpy(), t.a.double().cpu().numpy()
    # y = a·x + b: b̄ = Σ ȳ, ā = Σ ȳ·x + l̄/a
    ab = (Y * X).sum(axis=1) + LB.sum() / a
    bb = Y.sum(axis=1)
    assert rel(B.to_numpy(grads[0]["a"]), ab) <= 2e-5
    assert rel(B.to_numpy(grads[1]["a"]), bb) <= 2e-5


# ---- Float64 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("law", list(LAWS))
def test_float64(B, law, inverse):
    import torch

    rng = seed("f64", law, inverse)
    D, N = 37, 211
    lay = vec(B, LAWS[law], param(LAWS[law], D, rng), torch.float64)
    t = B.inverse(lay) if inverse else lay
    o = E.VecLayer(LAWS[law], lay.a.cpu().numpy())
    x, ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    xd = torch.from_numpy(x.T.copy()).cuda().t()
    y, lj = B.with_logabsdet_jacobian(t, xd)
    yo, ljo = (o.inverse if inverse else o.forward)(x)
    assert rel(y.cpu().numpy(), yo) <= 1e-12 and np.abs(lj.cpu().numpy() - ljo).max() <= 1e-12 * max(1, np.abs(ljo).max())
    xb, grads = B.chain_vjp(t, xd, torch.from_numpy(ybar.T.copy()).cuda().t(), torch.from_numpy(ljbar).cuda())
    xo, go = o.vjp(x, ybar, ljbar, inverse)
    assert rel(xb.cpu().numpy(), xo) <= 1e-12
    assert rel(grads[0][o.name].cpu().numpy(), go[o.name]) <= 1e-12


# ---- training -----------------------------------------------------------------------------------------------------------
def test_flow_fit_recovers_affine(B):
    """Flow(Shift(b) ∘ Scale(a), MvNormal(D)) fitted by Adam to y = μ* + σ* ⊙ z recovers μ* and σ*."""
    import torch

    D, N = 16, 1 << 16
    rng = seed("fit")
    mu_t, sg_t = rng.standard_normal(D), rng.uniform(0.5, 2.0, D)
    g = torch.Generator(device="cuda").manual_seed(3)
    z = torch.randn(N, D, device="cuda", generator=g).t()
    y = (torch.from_numpy(mu_t).float().cuda()[:, None] + torch.from_numpy(sg_t).float().cuda()[:, None] * z)
    y = y.t().contiguous().t()
    s, t = B.Scale(np.ones(D, f32)), B.Shift(np.zeros(D, f32))
    model = B.autograd.Flow(B.ComposedFunction(t, s), B.MvNormal(D))
    assert len(model.params) == 2
    opt = torch.optim.Adam(model.parameters(), lr=0.05)
    for _ in range(600):
        opt.zero_grad()
        loss = model.nll(y) / N
        loss.backward()
        opt.step()
    assert np.abs(np.abs(B.to_numpy(s.a)) - sg_t).max() <= 2e-2
    assert np.abs(B.to_numpy(t.a) - mu_t).max() <= 2e-2


def test_rsample_gradients(B):
    """Flow.rsample: ā, b̄ of Σ w⊙y + Σ c·log q against the reparameterisation gradient (z = (y − b)/a)."""
    import torch

    D, N = 24, 5000
    rng = seed("rsample")
    a, b = param(E.SCALE, D, rng), param(E.SHIFT, D, rng)
    s, t = vec(B, E.SCALE, a), vec(B, E.SHIFT, b)
    model = B.autograd.Flow(B.ComposedFunction(t, s), B.MvNormal(D))
    y, lq = model.rsample(N, seed=11)
    w = torch.from_numpy(rng.standard_normal((D, N)).astype(f32)).cuda()
    c = torch.from_numpy(rng.standard_normal(N).astype(f32)).cuda()
    ((w * y).sum() + (c * lq).sum()).backward()
    A, Bv = s.a.double().cpu().numpy(), t.a.double().cpu().numpy()
    Z = (y.detach().double().cpu().numpy() - Bv[:, None]) / A[:, None]
    W, C = w.double().cpu().numpy(), c.double().cpu().numpy()
    ga, gb = (W * Z).sum(axis=1) - C.sum() / A, W.sum(axis=1)
    pa, pb = model.params[1].grad, model.params[0].grad  # leaves in flatten order: Scale, then Shift
    if pa.data_ptr() != s.a.data_ptr():
        pa, pb = pb, pa
    assert rel(pa.double().cpu().numpy(), ga) <= 1e-4 and rel(pb.double().cpu().numpy(), gb) <= 1e-5


# ---- sampler ------------------------------------------------------------------------------------------------------------
def test_sampler_one_launch(B):
    D, n = 128, 10000
    rng = seed("rand")
    s, t = vec(B, E.SCALE, param(E.SCALE, D, rng)), vec(B, E.SHIFT, param(E.SHIFT, D, rng))
    pl = B.PlanarLayer(D)
    td = B.transformed(B.MvNormal(D), B.ComposedFunction(t, B.ComposedFunction(s, pl)))
    ys, qs = B.rand_logpdf(td, n, seed=5)
    n1 = launches(B)
    ye, qe = B.rand_logpdf(B.transformed(B.MvNormal(D), B.Composed(pl, stacked_eq(B, s), stacked_eq(B, t))), n, seed=5)
    assert n1 == 1 and launches(B) == 1
    assert np.array_equal(B.to_numpy(ys), B.to_numpy(ye)) and np.array_equal(B.to_numpy(qs), B.to_numpy(qe))
    assert np.array_equal(B.to_numpy(B.rand(td, n, seed=5)), B.to_numpy(ys))
