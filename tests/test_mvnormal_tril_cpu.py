"""CPU tests of the full-covariance MvNormal base: the float64 reference of tests/mvnormal_tril_oracle.py against scipy and
central differences, and the Python constructor rules of MvNormal(D, mu, sigma; cov, scale_tril)."""
import numpy as np
import pytest
import scipy.stats

import mvnormal_tril_oracle as T


@pytest.mark.parametrize("cond", [1.0, 1e3])
@pytest.mark.parametrize("D", [1, 2, 5, 64])
def test_oracle_logpdf_matches_scipy(D, cond):
    rng = np.random.default_rng(D)
    L = T.random_tril(rng, D, cond)
    mu = rng.standard_normal(D)
    x = mu[:, None] + L @ rng.standard_normal((D, 9))
    ref = scipy.stats.multivariate_normal(mean=mu, cov=L @ L.T, allow_singular=False).logpdf(x.T)
    np.testing.assert_allclose(T.logpdf(L, mu, x), np.atleast_1d(ref), rtol=1e-9, atol=1e-9)


def test_oracle_ignores_upper_triangle():
    rng = np.random.default_rng(7)
    L = T.random_tril(rng, 6)
    x = rng.standard_normal((6, 4))
    Lu = L + np.triu(rng.standard_normal((6, 6)), 1)
    np.testing.assert_array_equal(T.logpdf(Lu, None, x), T.logpdf(L, None, x))


@pytest.mark.parametrize("D", [1, 4, 7])
def test_oracle_vjp_central_differences(D):
    rng = np.random.default_rng(100 + D)
    N = 5
    L = T.random_tril(rng, D)
    mu = rng.standard_normal(D)
    x = rng.standard_normal((D, N))
    lb = rng.standard_normal(N)
    gx, gm, gL = T.logpdf_vjp(L, mu, x, lb)
    f = lambda L_, mu_, x_: float(lb @ T.logpdf(L_, mu_, x_))
    h = 1e-6
    num_x = np.zeros_like(x)
    for i in range(D):
        for n in range(N):
            e = np.zeros_like(x)
            e[i, n] = h
            num_x[i, n] = (f(L, mu, x + e) - f(L, mu, x - e)) / (2 * h)
    num_m = np.array([(f(L, mu + h * np.eye(D)[i], x) - f(L, mu - h * np.eye(D)[i], x)) / (2 * h) for i in range(D)])
    num_L = np.zeros((D, D))
    for i in range(D):
        for j in range(i + 1):
            e = np.zeros((D, D))
            e[i, j] = h
            num_L[i, j] = (f(L + e, mu, x) - f(L - e, mu, x)) / (2 * h)
    np.testing.assert_allclose(gx, num_x, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(gm, num_m, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(gL, num_L, rtol=1e-6, atol=1e-6)
    assert np.all(np.triu(gL, 1) == 0)


def test_oracle_sample_is_unwhiten():
    rng = np.random.default_rng(3)
    L = T.random_tril(rng, 5)
    mu = rng.standard_normal(5)
    z = rng.standard_normal((5, 3))
    y = T.sample(L, mu, z)
    np.testing.assert_allclose(np.linalg.solve(L, y - mu[:, None]), z, rtol=1e-12, atol=1e-12)


@pytest.fixture(scope="module")
def B():
    import bijectors_jl_b200 as B

    return B


def test_mvnormal_at_most_one_covariance(B):
    eye = np.eye(3)
    for kw in (dict(sigma=np.ones(3), cov=eye), dict(sigma=np.ones(3), scale_tril=eye), dict(cov=eye, scale_tril=eye),
               dict(sigma=np.ones(3), cov=eye, scale_tril=eye)):
        with pytest.raises(ValueError, match="at most one"):
            B.MvNormal(3, device="cpu", **kw)


def test_mvnormal_cov_not_posdef(B):
    bad = np.array([[1.0, 2.0], [2.0, 1.0]])
    with pytest.raises(B.PosDefException, match="not positive definite"):
        B.MvNormal(2, cov=bad, device="cpu")
    with pytest.raises(ValueError):  # PosDefException is a ValueError
        B.MvNormal(2, cov=-np.eye(2), device="cpu")


def test_mvnormal_cov_is_factorised(B):
    rng = np.random.default_rng(11)
    L = T.random_tril(rng, 4)
    d = B.MvNormal(4, mu=np.zeros(4), cov=L @ L.T, device="cpu")
    np.testing.assert_allclose(d.scale_tril.numpy(), L.astype(np.float32), rtol=1e-5, atol=1e-6)
    assert d._terminal_desc().kind == 9
    assert B.MvNormal(4, device="cpu")._terminal_desc().kind == 8
    with pytest.raises(ValueError, match="DimensionMismatch"):
        B.MvNormal(3, cov=L @ L.T, device="cpu")


def test_float64_factor_builds_a_float64_terminal_and_has_no_sampler(B):
    import torch

    L = np.tril(np.ones((3, 3))) + np.eye(3)
    d = B.MvNormal(3, mu=np.zeros(3), scale_tril=L, device="cpu", dtype=torch.float64)
    desc = d._terminal_desc()
    assert isinstance(desc, B._lib.LayerDesc64) and desc.kind == B._lib.MVNORMAL_TRIL
    assert d.scale_tril.dtype == torch.float64
    with pytest.raises(TypeError, match="no device sampler"):
        B.rand(d, 4, seed=1)
    with pytest.raises(TypeError, match="no device sampler"):
        B.rand(B.transformed(d, B.Composed()), 4, seed=1)
