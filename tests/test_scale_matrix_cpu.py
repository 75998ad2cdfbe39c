"""CPU tests of the dense Scale layer's float64 oracle (tests/scale_matrix_oracle.py), its header constants and the Python
descriptor: no GPU needed."""
import os

import numpy as np
import pytest

import scale_matrix_oracle as S


def _loss(A, x, yb, lb, inv):
    y, lj = (S.inverse if inv else S.forward)(A, x)
    return float(np.sum(yb * y) + np.sum(lb * lj))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D", [1, 3, 5])
def test_vjp_matches_central_differences(D, inv):
    rng = np.random.default_rng(10 * D + inv)
    N = 4
    A = S.well_conditioned(rng, D, 0.3)
    if D >= 3:
        A[[0, 1]] = A[[1, 0]]  # det A < 0
        A[0, 0] = 0.0  # and a zero where the first pivot would be: the determinant stays well away from 0
        assert abs(np.linalg.det(A)) > 0.5 and np.linalg.cond(A) < 10
    x = rng.standard_normal((D, N))
    yb = rng.standard_normal((D, N))
    lb = rng.standard_normal(N)
    xb, Ab = S.vjp(A, x, yb, lb, inverse=inv)
    h = 1e-6
    for i in range(D):
        for n in range(N):
            e = np.zeros_like(x)
            e[i, n] = h
            fd = (_loss(A, x + e, yb, lb, inv) - _loss(A, x - e, yb, lb, inv)) / (2 * h)
            assert abs(fd - xb[i, n]) <= 1e-6 * max(1.0, abs(fd)), (i, n)
    for i in range(D):
        for j in range(D):
            E = np.zeros_like(A)
            E[i, j] = h
            fd = (_loss(A + E, x, yb, lb, inv) - _loss(A - E, x, yb, lb, inv)) / (2 * h)
            assert abs(fd - Ab[i, j]) <= 1e-6 * max(1.0, abs(fd)), (i, j)


def test_vjp_without_cotangents():
    rng = np.random.default_rng(3)
    A = S.well_conditioned(rng, 4)
    x = rng.standard_normal((4, 6))
    for inv in (False, True):
        xb, Ab = S.vjp(A, x, None, None, inverse=inv)
        assert not xb.any() and not Ab.any()
        xb, Ab = S.vjp(A, x, None, np.ones(6), inverse=inv)
        assert not xb.any()
        assert np.allclose(Ab, (-6.0 if inv else 6.0) * np.linalg.inv(A).T)


def test_forward_inverse_and_negative_determinant():
    rng = np.random.default_rng(5)
    A = S.well_conditioned(rng, 6)
    A[[0, 1]] = A[[1, 0]]  # one row swap: det A < 0
    assert np.linalg.det(A) < 0
    x = rng.standard_normal((6, 9))
    y, lj = S.forward(A, x)
    xr, lji = S.inverse(A, y)
    assert np.allclose(xr, x) and np.allclose(lj, np.log(abs(np.linalg.det(A)))) and np.allclose(lji, -lj)


def test_header_declares_the_kind_and_its_envelope():
    from bijectors_jl_b200 import _lib

    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "b2b.h")).read()
    assert "#define B2B_SCALE_MATRIX 12" in hdr and _lib.SCALE_MATRIX == 12
    assert "#define B2B_SCALE_MATRIX_MAX_D 256" in hdr and _lib.SCALE_MATRIX_MAX_D == 256
    assert "#define B2B_SCALE_MATRIX 10" not in hdr  # 10 stays an invalid kind


def test_descriptor_and_slot_shapes():
    import torch

    import bijectors_jl_b200 as B
    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200.autograd import _trainable_tensors
    from bijectors_jl_b200.interface import _SLOT_NAMES, _leaf_grads, _slot_shape, _trainable_slots

    A = np.arange(9, dtype=np.float32).reshape(3, 3)
    s = B.Scale(A, device="cpu")
    assert s.dense and np.array_equal(s.a.numpy(), A)
    assert np.array_equal(s._A.numpy(), A.T)  # column-major storage: Aᵀ row-major
    (d,) = s._descs(False, 3)
    assert d.kind == _lib.SCALE_MATRIX and d.inverse == 0 and d.p0 == s._A.data_ptr()
    assert not any(getattr(d, f) for f in ("p1", "p2", "p3", "i0", "i1", "n0", "n1", "n2", "n3"))
    (di,) = B.inverse(s)._descs(False, 3)
    assert di.kind == _lib.SCALE_MATRIX and di.inverse == 1
    assert _SLOT_NAMES[_lib.SCALE_MATRIX] == ("a",) and _trainable_slots(d) == [0] and _slot_shape(d, 0, 3) == (3, 3)
    assert _trainable_tensors(s)[0] is s._A and _trainable_tensors(B.inverse(s))[0] is s._A
    g = torch.arange(9.0).reshape(3, 3)  # a cotangent in storage layout
    assert torch.equal(_leaf_grads([d], [1], {(0, 0): g})[0]["a"], g.t())
    with pytest.raises(ValueError):
        s._descs(False, 4)
    with pytest.raises(TypeError):
        B.Scale(A, device="cpu", dtype=torch.float64)
    with pytest.raises(TypeError):
        s._descs(False, 3, torch.float64)
    with pytest.raises(ValueError):
        B.Scale(np.zeros((2, 3)), device="cpu")


def test_equality_and_scalar_scale_unchanged():
    import bijectors_jl_b200 as B
    from bijectors_jl_b200 import _lib

    A = np.eye(2, dtype=np.float32) * 2
    assert B.Scale(A, device="cpu") == B.Scale(A.copy(), device="cpu")
    assert B.Scale(A, device="cpu") != B.Scale(A * 3, device="cpu")
    assert B.Scale(A, device="cpu") != B.Scale(2.0) and B.Scale(2.0) == B.Scale(2.0)
    s = B.Scale(2.5)
    assert not s.dense and s.a == 2.5 and s.code == _lib.EW_SCALE
    with pytest.raises(B.B2BError):
        B.Stacked([B.Scale(A, device="cpu")], [(1, 2)], device="cpu")
