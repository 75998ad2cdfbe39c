"""CPU tests of the spline coupling reference (tests/spline_coupling_oracle.py) and of the host-side pieces of
B2B_COUPLING_RQS: the oracle's reverse mode against central differences, its log-Jacobian against log|det J| of a
finite-difference Jacobian, the inverse, the constructor's shape errors and the descriptor fields."""
import numpy as np
import pytest

import spline_coupling_oracle as S


def _case(rng, D, idx1, idx2, K, scale=0.7):
    J = 3 * K - 1
    Wm = rng.standard_normal((J * len(idx1), len(idx2))) * scale
    c = rng.standard_normal(J * len(idx1)) * 0.5
    return Wm, c


def _fd(f, a, h=1e-6):
    g = np.zeros_like(a)
    for i in np.ndindex(a.shape):
        p, m = a.copy(), a.copy()
        p[i] += h
        m[i] -= h
        g[i] = (f(p) - f(m)) / (2 * h)
    return g


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("K", [2, 5])
def test_vjp_matches_central_differences(inv, K):
    rng = np.random.default_rng(10 * K + inv)
    D, N, Bv = 6, 4, 2.0
    idx1, idx2 = [2, 5, 1], [6, 3]  # row 4 is an x₃ row
    Wm, c = _case(rng, D, idx1, idx2, K)
    x = rng.uniform(-2.3, 2.3, (D, N))
    x[1, 0] = 2.5  # outside the box: the identity, no knot cotangent
    yb, lb = rng.standard_normal((D, N)), rng.standard_normal(N)
    f = S.inverse if inv else S.forward

    def loss(x_, W_, c_):
        y, lj = f(idx1, idx2, W_, c_, K, Bv, x_)
        return float(np.sum(y * yb) + np.sum(lj * lb))

    xb, Wb, cb = S.vjp(idx1, idx2, Wm, c, K, Bv, x, yb, lb, inverse=inv)
    for got, want in ((xb, _fd(lambda a: loss(a, Wm, c), x)), (Wb, _fd(lambda a: loss(x, a, c), Wm)),
                      (cb, _fd(lambda a: loss(x, Wm, a), c))):
        assert np.abs(got - want).max() <= 1e-6 * max(1.0, np.abs(want).max())


def test_vjp_on_the_box_edge_is_the_identity():
    """An element on the box edge (|x| = B exactly after the knots' own rounding) is the identity: ȳ passes through and it
    adds no cotangent to W or c."""
    rng = np.random.default_rng(2)
    K, Bv = 3, 1.5
    idx1, idx2 = [1], [2]
    Wm, c = _case(rng, 2, idx1, idx2, K)
    x = np.array([[1.5, -1.5, 0.3], [0.2, -0.4, 0.1]])
    yb = np.array([[1.0, 2.0, 0.0], [0.0, 0.0, 0.0]])
    for inv in (False, True):
        xb, Wb, cb = S.vjp(idx1, idx2, Wm, c, K, Bv, x, yb, np.zeros(3), inverse=inv)
        assert xb[0, 0] == 1.0 and xb[0, 1] == 2.0
        assert np.all(xb[1] == 0) and np.all(Wb == 0) and np.all(cb == 0)


def test_logjac_is_log_det_of_the_jacobian():
    rng = np.random.default_rng(4)
    D, K, Bv = 5, 4, 2.0
    idx1, idx2 = [1, 4], [2, 5]
    Wm, c = _case(rng, D, idx1, idx2, K)
    x = rng.uniform(-1.8, 1.8, D)
    for f in (S.forward, S.inverse):
        def col(v):
            return f(idx1, idx2, Wm, c, K, Bv, v[:, None])[0][:, 0]

        Jm = np.stack([(col(x + h) - col(x - h)) / 2e-6 for h in np.eye(D) * 1e-6], axis=1)
        lj = f(idx1, idx2, Wm, c, K, Bv, x[:, None])[1][0]
        assert abs(np.log(abs(np.linalg.det(Jm))) - lj) < 1e-6


def test_inverse_of_forward():
    rng = np.random.default_rng(6)
    D, N, K, Bv = 7, 30, 6, 3.0
    idx1, idx2 = [7, 1, 3], [2, 4, 6]
    Wm, c = _case(rng, D, idx1, idx2, K)
    x = rng.uniform(-3.2, 3.2, (D, N))
    y, lj = S.forward(idx1, idx2, Wm, c, K, Bv, x)
    xr, ljr = S.inverse(idx1, idx2, Wm, c, K, Bv, y)
    # float64 round trip; the inverse's quadratic root loses a few digits in steep bins
    np.testing.assert_allclose(xr, x, atol=1e-8, rtol=0)
    np.testing.assert_allclose(ljr, -lj, atol=1e-8, rtol=0)
    assert np.array_equal(y[[1, 3, 4, 5]], x[[1, 3, 4, 5]])


def test_zero_W_gives_the_plain_spline():
    from oracle import oracle_np as O

    rng = np.random.default_rng(8)
    K, Bv = 5, 2.0
    idx1, idx2 = [1, 2], [3]
    _, c = _case(rng, 3, idx1, idx2, K)
    Wm = np.zeros(((3 * K - 1) * 2, 1))
    x = rng.uniform(-2, 2, (3, 9))
    y, lj = S.forward(idx1, idx2, Wm, c, K, Bv, x)
    rw, rh, rd = S.raw_params(Wm, c, np.zeros(1), K)
    ys, ljs = O.rqs_forward(*O.rqs_params(rw, rh, rd, Bv), x[:2])
    assert np.array_equal(y[:2], ys) and np.allclose(lj, ljs, rtol=0, atol=1e-14)


def test_conditioner_shapes_and_descriptor():
    import torch

    import bijectors_jl_b200 as B
    from bijectors_jl_b200 import _lib

    K, n1, n2 = 4, 3, 2
    J = 3 * K - 1
    with pytest.raises(ValueError):
        B.SplineConditioner(np.zeros((J * n1 + 1, n2), np.float32), K=K, B=1.0, device="cpu")
    with pytest.raises(ValueError):
        B.SplineConditioner(np.zeros((J * n1, n2), np.float32), np.zeros(J * n1 - 1, np.float32), K=K, B=1.0, device="cpu")
    with pytest.raises(ValueError):
        B.SplineConditioner(np.zeros((J * n1, n2), np.float32), K=K, B=0.0, device="cpu")
    with pytest.raises(TypeError):
        B.SplineConditioner(np.zeros((J * n1, n2)), K=K, B=1.0, device="cpu", dtype=torch.float64)
    W = np.arange(J * n1 * n2, dtype=np.float32).reshape(J * n1, n2)
    cond = B.SplineConditioner(W, np.ones(J * n1, np.float32), K=K, B=2.5, device="cpu")
    assert (cond.n1, cond.n2, cond.K, cond.B) == (n1, n2, K, 2.5)
    assert np.array_equal(cond.W.numpy().T, W)  # column-major storage
    mask = B.PartitionMask(7, [2, 4, 6], [1, 7])
    with pytest.raises(ValueError):
        B.Coupling(cond, B.PartitionMask(7, [2, 4], [1, 7]))
    cl = B.Coupling(cond, mask)
    d = cl._descs(True, 7)[0]
    assert (d.kind, d.inverse, d.n0, d.n1, d.n2, d.n3) == (_lib.COUPLING_RQS, 1, n1, n2, K, 0) and d.f0 == 2.5
    assert d.p0 == cond.W.data_ptr() and d.p1 == cond.c.data_ptr() and d.p2 is None and d.p3 is None
    assert d.i0 == cl._idx1.data_ptr() and d.i1 == cl._idx2.data_ptr()
    assert cl._idx1.tolist() == [1, 3, 5] and cl._idx2.tolist() == [0, 6]
    nc = B.Coupling(B.SplineConditioner(W, K=K, B=2.5, device="cpu"), mask)._descs(False, 7)[0]
    assert nc.p1 is None
    assert _lib.COUPLING_RQS == 11 and B.coupling(cl) is cond
    assert cl == B.Coupling(cond.to("cpu"), mask)


def test_header_declares_the_kind_and_its_envelope():
    import os

    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "b2b.h")).read()
    assert "#define B2B_COUPLING_RQS 11" in hdr
    assert "#define B2B_COUPLING_RQS_MAX_N 128" in hdr and "#define B2B_COUPLING_RQS_MAX_K 16" in hdr
    assert "#define B2B_COUPLING_RQS_MAX_D 1024" in hdr
    assert "#define B2B_" not in "".join(line for line in hdr.splitlines() if " 10 " in line and line.startswith("#define"))
