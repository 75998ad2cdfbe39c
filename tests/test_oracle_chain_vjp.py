"""CPU checks of the float64 reverse-mode restatements in tests/chain_vjp_oracle.py against central finite differences:
every Stacked law in both directions (Truncated inside and outside its box, with one-sided and infinite bounds), Permute,
the terminal MvNormal and mixed chains -- including a chain of every layer kind closed by either terminal."""
import numpy as np
import pytest

import chain_vjp_oracle as V
import coupling_mlp_oracle as M
import mvnormal_tril_oracle as T
import scale_matrix_oracle as SM
import spline_coupling_oracle as SC
from oracle import oracle_np as O

EW = O.EW
INF = float("inf")
LAWS = [
    ((EW.IDENTITY, 0.0), (-2, 2)), ((EW.EXP, 0.0), (-2, 2)), ((EW.LOG, 0.0), (0.3, 3)), ((EW.SHIFT, 0.7), (-2, 2)),
    ((EW.SCALE, -1.7), (-2, 2)), ((EW.LEAKY_RELU, 0.1), (-2, 2)), ((EW.LOGIT, -1.0, 3.0), (-0.9, 2.9)),
    ((EW.TRUNCATED, -1.0, 3.0), (-2, 4)), ((EW.TRUNCATED, -1.0, INF), (-2, 4)), ((EW.TRUNCATED, -INF, 3.0), (-2, 4)),
    ((EW.TRUNCATED, -INF, INF), (-2, 4)),
]


def _objective(fn, ybar, ljbar):
    def f(x):
        y, lj = fn(x)
        return float(np.sum(ybar * y) + np.sum(ljbar * lj))
    return f


def _fd(f, x, h=1e-6):
    g = np.zeros_like(x)
    for idx in np.ndindex(x.shape):
        xp, xm = x.copy(), x.copy()
        xp[idx] += h
        xm[idx] -= h
        g[idx] = (f(xp) - f(xm)) / (2 * h)
    return g


def _law_domain(op, inverse, lohi, rng, shape):
    x = rng.uniform(lohi[0], lohi[1], shape)
    if inverse:  # inputs of the inverse are outputs of the law
        if op[0] == EW.LOG:
            x = rng.uniform(-2, 1, shape)
        elif op[0] in (EW.LOGIT, EW.TRUNCATED) or op[0] == EW.EXP:
            x = rng.uniform(-2, 2, shape) if op[0] != EW.EXP else rng.uniform(0.3, 3, shape)
    return x


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("law", range(len(LAWS)))
def test_stacked_vjp_matches_finite_differences(law, inverse):
    op, lohi = LAWS[law]
    rng = np.random.default_rng(law * 2 + inverse)
    D, N = 3, 5
    x = _law_domain(op, inverse, lohi, rng, (D, N))
    x[np.abs(x) < 1e-3] += 0.01  # keep clear of LeakyReLU's kink
    if op[0] == EW.TRUNCATED and not inverse:  # a clamped point has an infinite log-Jacobian: see the test below
        lo, hi = op[1], op[2]
        x = np.clip(x, lo + 0.05 if np.isfinite(lo) else -np.inf, hi - 0.05 if np.isfinite(hi) else np.inf)
    ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal(N)
    ranges = [(1, D)]
    fn = (lambda z: O.stacked_inverse([op], ranges, z)) if inverse else (lambda z: O.stacked_forward([op], ranges, z))
    got = V.stacked_vjp([op], ranges, x, ybar, ljbar, inverse=inverse)
    np.testing.assert_allclose(got, _fd(_objective(fn, ybar, ljbar), x), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("lo,hi", [(-1.0, 3.0), (-1.0, INF), (-INF, 3.0)])
def test_truncated_forward_is_flat_outside_the_box(lo, hi):
    # AD of _clamp: points outside [lb, ub] do not move the output (nor its log-Jacobian)
    x = np.array([[-3.0, 5.0, 0.5]])
    got = V.stacked_vjp([(EW.TRUNCATED, lo, hi)], [(1, 1)], x, np.full((1, 3), 2.0), np.ones(3))
    assert got[0, 2] != 0
    if np.isfinite(lo):
        assert got[0, 0] == 0
    if np.isfinite(hi):
        assert got[0, 1] == 0


@pytest.mark.parametrize("inverse", [False, True])
def test_permute_vjp_matches_finite_differences(inverse):
    rng = np.random.default_rng(7)
    A = O.permute_matrix_from_indices([3, 1, 4, 2])
    x, ybar = rng.standard_normal((4, 3)), rng.standard_normal((4, 3))
    fn = (lambda z: O.permute_inverse(A, z)) if inverse else (lambda z: O.permute_forward(A, z))
    np.testing.assert_allclose(V.permute_vjp(A, ybar, inverse), _fd(_objective(fn, ybar, np.zeros(3)), x), atol=1e-7)


@pytest.mark.parametrize("given", ["none", "mu", "sigma", "both"])
def test_mvnormal_vjp_matches_finite_differences(given):
    rng = np.random.default_rng(3)
    D, N = 4, 3
    mu = rng.standard_normal(D) if given in ("mu", "both") else None
    sigma = rng.uniform(0.5, 2, D) if given in ("sigma", "both") else None
    x, lb = rng.standard_normal((D, N)), rng.standard_normal(N)
    xb, mb, sb = V.mvnormal_diag_logpdf_vjp(mu, sigma, x, lb)
    f = lambda z, m=mu, s=sigma: float(np.sum(lb * O.mvnormal_diag_logpdf(m, s, z)))
    np.testing.assert_allclose(xb, _fd(f, x), rtol=1e-6, atol=1e-7)
    m0 = np.zeros(D) if mu is None else mu
    s0 = np.ones(D) if sigma is None else sigma
    np.testing.assert_allclose(mb, _fd(lambda m: float(np.sum(lb * O.mvnormal_diag_logpdf(m, s0, x))), m0), rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(sb, _fd(lambda s: float(np.sum(lb * O.mvnormal_diag_logpdf(m0, s, x))), s0), rtol=1e-6, atol=1e-7)


def _mixed_chain(rng, D):
    w, u = rng.standard_normal(D) * 0.5, rng.standard_normal(D) * 0.5
    ops = [(EW.EXP, 0.0), (EW.SCALE, -1.3), (EW.TRUNCATED, -4.0, 4.0)]
    ranges = [(1, 1), (2, 2), (3, D)]
    layers = [O.Layer("planar", dict(w=w, u=u, b=np.array([0.2]))),
              O.Layer("permute", dict(A=O.permute_matrix_from_indices(list(rng.permutation(D) + 1)))),
              O.Layer("stacked", dict(ops=ops, ranges=ranges)),
              O.Layer("radial", dict(alpha_raw=np.array([0.3]), beta=np.array([0.4]), z0=rng.standard_normal(D) * 0.3))]
    return layers


@pytest.mark.parametrize("terminal", [False, True])
def test_chain_vjp_matches_finite_differences(terminal):
    rng = np.random.default_rng(11)
    D, N = 4, 3
    layers = _mixed_chain(rng, D)
    flags = [False, True, False, True]
    x = rng.standard_normal((D, N)) * 0.5
    mu, sigma = rng.standard_normal(D) * 0.2, rng.uniform(0.7, 1.4, D)
    ybar = None if terminal else rng.standard_normal((D, N))
    lb = rng.standard_normal(N)

    def f(z):
        y, lj = V.chain_logjac(layers, flags, z, mu, sigma, terminal)
        return float((0 if ybar is None else np.sum(ybar * y)) + np.sum(lb * lj))

    xb, grads, base = V.chain_vjp(layers, flags, x, ybar, lb, mu, sigma, terminal)
    np.testing.assert_allclose(xb, _fd(f, x), rtol=1e-5, atol=1e-6)
    # parameter cotangents: planar w and radial z_0 by finite differences through the layer objects
    for l, key, name in ((0, "w", "w"), (3, "z0", "z_0")):
        p0 = layers[l].params[key].copy()

        def fp(v, l=l, key=key):
            layers[l].params[key] = v
            try:
                return f(x)
            finally:
                layers[l].params[key] = p0
        np.testing.assert_allclose(grads[l][name], _fd(fp, p0), rtol=1e-5, atol=1e-6)
    if terminal:
        assert set(base) == {"μ", "σ"}


# ---- chains of every layer kind, closed by either terminal ------------------------------------------------------------------
NEW_KIND_FLAGS = [False, True, False, True, False, True, False, False, True, False, True, True]


def _every_kind_params(rng, D=6):
    """Parameters of the chain _every_kind_layers builds (a dict of float64 arrays, perturbed by the finite differences)."""
    K = 4
    r = lambda *s: rng.standard_normal(s)  # noqa: E731
    return dict(perm=rng.permutation(D) + 1, rw=r(D, K) * 0.5, rh=r(D, K) * 0.5, rd=r(D, K - 1) * 0.5,
                bn_b=r(D) * 0.1, bn_logs=r(D) * 0.1, bn_m=r(D) * 0.1, bn_v=rng.uniform(0.5, 1.5, D),
                aW=r(4, 3) * 0.2, ac=r(4) * 0.1, sW=r((3 * K - 1) * 2, 4) * 0.3, sc=r((3 * K - 1) * 2) * 0.3,
                A=np.eye(D) + 0.3 * r(D, D) / np.sqrt(D), m1W1=r(5, 3) * 0.5, m1c1=r(5) * 0.3, m1W2=r(6, 5) * 0.2,
                m1c2=r(6) * 0.2, m2W1=r(4, 3) * 0.5, m2W2=r(4, 4) * 0.2, pw=r(D) * 0.4, pu=r(D) * 0.4, pb=r(1),
                qw=r(D) * 0.4, qu=r(D) * 0.4, qb=r(1), ra=r(1), rb=r(1), rz=r(D) * 0.3)


def _every_kind_layers(p, K=4):
    """Stacked -> Inverse(Permute) -> RQS -> Inverse(BatchNorm) -> affine Coupling (index lists, an x₃ row) ->
    Inverse(spline Coupling) -> Scale -> MLP Coupling (tanh) -> Inverse(MLP Coupling, LeakyReLU, no biases) -> planar ->
    Inverse(planar) -> Inverse(radial), at D = 6: every layer kind of the chain, flags NEW_KIND_FLAGS."""
    ops = [(EW.EXP, 0.0), (EW.SCALE, -1.3), (EW.SHIFT, 0.4)]
    W, H, Dv = O.rqs_params(p["rw"], p["rh"], p["rd"], 3.0)
    return [O.Layer("stacked", dict(ops=ops, ranges=[(1, 1), (2, 3), (4, 6)])),
            O.Layer("permute", dict(A=O.permute_matrix_from_indices(list(p["perm"])))),
            O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv)),
            O.Layer("batchnorm", dict(bn=O.BatchNormParams(b=p["bn_b"], logs=p["bn_logs"], m=p["bn_m"], v=p["bn_v"],
                                                           eps=1e-5))),
            O.Layer("coupling_affine", dict(idx1=np.array([2, 5]), idx2=np.array([1, 3, 6]), W=p["aW"], c=p["ac"])),
            SC.SplineLayer([1, 4], [2, 3, 5, 6], p["sW"], p["sc"], K, 3.0),
            SM.ScaleLayer(p["A"]),
            M.MLPLayer([3, 6, 1], [2, 4, 5], p["m1W1"], p["m1c1"], p["m1W2"], p["m1c2"], "tanh"),
            M.MLPLayer([4, 5], [1, 2, 3], p["m2W1"], None, p["m2W2"], None, "leaky_relu", 0.2),
            O.Layer("planar", dict(w=p["pw"], u=p["pu"], b=p["pb"])),
            O.Layer("planar", dict(w=p["qw"], u=p["qu"], b=p["qb"])),
            O.Layer("radial", dict(alpha_raw=p["ra"], beta=p["rb"], z0=p["rz"]))]


# (layer, cotangent name, parameter key) checked by finite differences: every parameter of the spline, Scale and MLP layers
NEW_KIND_PARAMS = [(5, "W", "sW"), (5, "c", "sc"), (6, "a", "A"), (7, "W1", "m1W1"), (7, "c1", "m1c1"), (7, "W2", "m1W2"),
                   (7, "c2", "m1c2"), (8, "W1", "m2W1"), (8, "W2", "m2W2"), (4, "W", "aW"), (9, "w", "pw")]


@pytest.mark.parametrize("terminal", ["none", "diag", "tril"])
def test_every_kind_chain_matches_finite_differences(terminal):
    rng = np.random.default_rng(23 + len(terminal))
    D, N = 6, 4
    p = _every_kind_params(rng, D)
    x = rng.standard_normal((D, N)) * 0.5
    mu, sigma = rng.standard_normal(D) * 0.2, rng.uniform(0.7, 1.4, D)
    L = T.random_tril(rng, D)
    ybar = rng.standard_normal((D, N)) if terminal != "tril" else None
    lb = rng.standard_normal(N)
    kw = dict(none={}, diag=dict(mu=mu, sigma=sigma, terminal=True), tril=dict(mu=mu, scale_tril=L))[terminal]

    def f(z, q=p, **over):
        y, lj = V.chain_logjac(_every_kind_layers(q), NEW_KIND_FLAGS, z, **{**kw, **over})
        return float((0 if ybar is None else np.sum(ybar * y)) + np.sum(lb * lj))

    xb, grads, base = V.chain_vjp(_every_kind_layers(p), NEW_KIND_FLAGS, x, ybar, lb, **kw)
    np.testing.assert_allclose(xb, _fd(f, x), rtol=1e-5, atol=1e-6)
    for l, name, key in NEW_KIND_PARAMS:
        fp = lambda v, key=key: f(x, {**p, key: v})  # noqa: E731
        np.testing.assert_allclose(grads[l][name], _fd(fp, p[key]), rtol=1e-5, atol=1e-6, err_msg=f"{l} {name}")
    if terminal == "diag":
        assert set(base) == {"μ", "σ"}
        np.testing.assert_allclose(base["σ"], _fd(lambda s: f(x, sigma=s), sigma), rtol=1e-5, atol=1e-6)
    if terminal == "tril":
        assert set(base) == {"μ", "L"}
        Lfd = np.tril(_fd(lambda m: f(x, scale_tril=m), L))
        np.testing.assert_allclose(base["L"], Lfd, rtol=1e-5, atol=1e-6)
    if terminal != "none":
        np.testing.assert_allclose(base["μ"], _fd(lambda m: f(x, mu=m), mu), rtol=1e-5, atol=1e-6)


def test_new_kind_vjps_evaluate_in_the_batch_dtype():
    """The spline, Scale and MLP layers' .vjp follow x's dtype, so that chain_vjp(..., dtype=float32) is a float32 result
    (the own-error term of the parity gates)."""
    rng = np.random.default_rng(29)
    D, N = 6, 5
    p = _every_kind_params(rng, D)
    x = rng.standard_normal((D, N)) * 0.5
    lb = rng.standard_normal(N)
    layers = _every_kind_layers(p)
    for l in (5, 6, 7, 8):
        for dt in (np.float32, np.float64):
            xb, g = V._layer_vjp(layers[l], NEW_KIND_FLAGS[l], x.astype(dt), np.ones((D, N), dt), lb.astype(dt))
            assert xb.dtype == dt and all(np.asarray(v).dtype == dt for v in g.values()), (l, dt)
    L = T.random_tril(rng, D)
    o64 = V.chain_vjp(layers[:9], NEW_KIND_FLAGS[:9], x, None, lb, scale_tril=L)
    o32 = V.chain_vjp(layers[:9], NEW_KIND_FLAGS[:9], x, None, lb, scale_tril=L, dtype=np.float32)
    assert o64[0].dtype == np.float64 and o32[0].dtype == np.float32 and o32[2]["L"].dtype == np.float32
    assert 0 < np.linalg.norm(o32[0] - o64[0]) <= 1e-4 * np.linalg.norm(o64[0])
