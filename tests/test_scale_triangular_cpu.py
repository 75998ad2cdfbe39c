"""CPU tests of the triangular Scale layer, B2B_SCALE_TRIANGULAR: the float64 oracle against central differences, the
constants of the header, the Python binding and the Julia shim, the status codes and workspace sizes of the host paths
(N = 0 calls and workspace queries), and the Python layer.  No GPU needed."""
import ctypes
import os
import re

import numpy as np
import pytest

import scale_triangular_oracle as S

ROOT = os.path.join(os.path.dirname(__file__), "..")


@pytest.fixture(scope="module")
def B():
    import bijectors_jl_b200 as B

    return B


# ---- the oracle -------------------------------------------------------------------------------------------------------
def _loss(T, upper, unit, x, yb, lb, inv):
    y, lj = (S.inverse if inv else S.forward)(T, upper, unit, x)
    return float(np.sum(yb * y) + np.sum(lb * lj))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("upper,unit", S.FORMS)
def test_vjp_matches_central_differences(upper, unit, inv):
    rng = np.random.default_rng(4 * upper + 2 * unit + inv)
    D, N, h = 5, 4, 1e-6
    T = S.random_tri(rng, D, upper, unit, np.float64)
    x, yb, lb = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    xb, Tb = S.vjp(T, upper, unit, x, yb, lb, inverse=inv)
    for i in range(D):
        for n in range(N):
            e = np.zeros_like(x)
            e[i, n] = h
            fd = (_loss(T, upper, unit, x + e, yb, lb, inv) - _loss(T, upper, unit, x - e, yb, lb, inv)) / (2 * h)
            assert abs(fd - xb[i, n]) <= 1e-6 * max(1.0, abs(fd)), (i, n)
    P = S.mask(D, upper, unit)
    for i in range(D):
        for j in range(D):
            E = np.zeros_like(T)
            E[i, j] = h
            fd = (_loss(T + E, upper, unit, x, yb, lb, inv) - _loss(T - E, upper, unit, x, yb, lb, inv)) / (2 * h)
            assert abs(fd - Tb[i, j]) <= 1e-6 * max(1.0, abs(fd)), (i, j)
            if not P[i, j]:  # an entry the view does not read: no effect, and exactly 0 in T̄
                assert fd == 0.0 and Tb[i, j] == 0.0


def test_oracle_matches_dense_algebra():
    rng = np.random.default_rng(9)
    D = 7
    for upper, unit in S.FORMS:
        T = S.random_tri(rng, D, upper, unit, np.float64)
        M = S.view(T, upper, unit)
        x = rng.standard_normal((D, 3))
        y, lj = S.forward(T, upper, unit, x)
        assert np.allclose(y, M @ x) and np.allclose(lj, np.linalg.slogdet(M)[1])
        xr, lji = S.inverse(T, upper, unit, y)
        assert np.allclose(xr, x) and np.allclose(lji, -lj)
        assert np.linalg.cond(M) < 20


# ---- constants ----------------------------------------------------------------------------------------------------------
def test_constants_agree(B):
    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    jl = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()
    assert int(re.search(r"#define B2B_SCALE_TRIANGULAR (\d+)", hdr).group(1)) == B._lib.SCALE_TRIANGULAR == 18
    assert int(re.search(r"#define B2B_SCALE_TRIANGULAR_MAX_D (\d+)", hdr).group(1)) == B._lib.SCALE_TRIANGULAR_MAX_D == 256
    assert int(re.search(r"const SCALE_TRIANGULAR = Int32\((\d+)\)", jl).group(1)) == 18
    assert int(re.search(r"const SCALE_TRIANGULAR_MAX_D = (\d+)", jl).group(1)) == 256
    kinds = [int(v) for v in re.findall(r"#define B2B_[A-Z_]+ (\d+)\s+/\*", hdr)]
    assert 18 in kinds and 10 not in kinds  # 10 stays an invalid kind


# ---- status codes and workspace sizes through the host paths -------------------------------------------------------------
def descs(B, D=8, n0=0, n1=0, inverse=0, p0=0x1000, f64=False, extra=()):
    d = (B._lib.LayerDesc64 if f64 else B._lib.LayerDesc)()
    d.kind, d.inverse, d.n0, d.n1, d.p0 = B._lib.SCALE_TRIANGULAR, inverse, n0, n1, p0
    return (type(d) * (1 + len(extra)))(d, *extra)


def vjp_status(B, arr, D, bars=None, f64=False):
    fn = B.lib().b2b_chain_vjp_f64 if f64 else B.lib().b2b_chain_vjp_f32
    L = len(arr)
    pb = None
    if bars is not None:
        ptrs = (ctypes.c_void_p * (4 * L))(*bars)
        pb = ctypes.cast(ptrs, ctypes.c_void_p)
    return fn(arr, L, 0x2000, None, None, 0x3000, pb, D, 0, D, D, D, None, 0, None)


def al256(b):
    return (b + 255) & ~255


def test_status_codes(B):
    lib, L_ = B.lib(), B._lib
    for f64 in (False, True):
        assert vjp_status(B, descs(B, f64=f64), 8, f64=f64) == L_.B2B_OK
        for n0, n1 in ((2, 0), (0, 2), (-1, 0), (0, -1)):
            assert vjp_status(B, descs(B, n0=n0, n1=n1, f64=f64), 8, f64=f64) == L_.B2B_EINVAL
        assert vjp_status(B, descs(B, p0=None, f64=f64), 8, f64=f64) == L_.B2B_EINVAL
        for slot in (1, 2, 3):
            bars = [None] * 4
            bars[slot] = 0x4000
            assert vjp_status(B, descs(B, f64=f64), 8, bars, f64=f64) == L_.B2B_EUNSUPPORTED, slot
    # the Float32 envelope: D <= 256, refused past it with workspace 0
    for inv in (0, 1):
        a = descs(B, D=257, inverse=inv)
        assert vjp_status(B, a, 257) == L_.B2B_EUNSUPPORTED
        assert lib.b2b_chain_workspace_bytes(a, 1, 257, 1000, 1, 0) == 0 and lib.b2b_workspace_bytes(a, 257, 1000) == 0
        assert lib.b2b_chain_vjp_workspace_bytes(a, 1, 257, 1000) == 0
        assert lib.b2b_chain_workspace_bytes(descs(B, inverse=inv), 1, 256, 1000, 1, 0) > 0
    # Float64: D <= 2048
    assert vjp_status(B, descs(B, f64=True), 2048, f64=True) == L_.B2B_OK
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, f64=True), 1, 2048, 100) > 0
    assert vjp_status(B, descs(B, f64=True), 2049, f64=True) == L_.B2B_EUNSUPPORTED
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, f64=True), 1, 2049, 100) == 0
    # refusals give workspace 0
    assert lib.b2b_chain_vjp_workspace_bytes(descs(B, n0=2), 1, 8, 1000) == 0
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, n1=3, f64=True), 1, 8, 1000) == 0


def test_workspace_formulas(B):
    """The chain workspace holds [M (4·D² B)][log|det T| (8 B)], each rounded up to 256, + 256; a chain holding dense and
    triangular Scale layers one region of the larger; the reverse mode adds P·D² floats and 2·D² + 1 doubles, P the column
    chunks of G."""
    lib, L_ = B.lib(), B._lib
    for D in (1, 5, 64, 200, 256):
        tri = al256(4 * D * D) + al256(8) + 256
        dense = al256(8 * D * D) + al256(4 * D * D) + al256(4 * D) + al256(8) + 256
        for inv in (0, 1):
            assert lib.b2b_chain_workspace_bytes(descs(B, inverse=inv), 1, D, 1000, 1, 0) == tri
            assert lib.b2b_workspace_bytes(descs(B, inverse=inv), D, 1000) == tri
        dm = L_.LayerDesc()
        dm.kind, dm.p0 = L_.SCALE_MATRIX, 0x1000
        assert lib.b2b_chain_workspace_bytes(descs(B, extra=(dm,)), 2, D, 1000, 1, 0) == dense
        for N, P in ((1, 1), (4096, 1), (5000, 2), (1 << 20, 64)):
            want = tri + al256(4 * P * D * D) + 2 * al256(8 * D * D) + al256(8)
            got = lib.b2b_chain_vjp_workspace_bytes(descs(B), 1, D, N)
            # + the chain reverse mode's two D x N cotangent buffers and its alignment slack
            assert got == want + 2 * al256(4 * D * N) + 256, (D, N, got, want)


def test_mixed_chains_size_and_refuse_together(B):
    """Inside chains with planar, coupling and MvNormal layers the queries are 0 exactly when a layer is refused."""
    lib, L_ = B.lib(), B._lib
    D, N = 64, 5000

    def chain(n0=0):
        pl, cp, mv = L_.LayerDesc(), L_.LayerDesc(), L_.LayerDesc()
        pl.kind, pl.p0, pl.p1, pl.p2 = L_.PLANAR, 0x1000, 0x1100, 0x1200
        cp.kind, cp.n0, cp.n1, cp.n2, cp.n3, cp.p0 = L_.COUPLING_AFFINE, 32, 32, 0, 32, 0x1300
        mv.kind = L_.MVNORMAL_DIAG
        t = descs(B, n0=n0)[0]
        return (L_.LayerDesc * 4)(pl, t, cp, mv)

    assert lib.b2b_chain_workspace_bytes(chain(), 4, D, N, 1, 0) > 0
    assert lib.b2b_chain_vjp_workspace_bytes(chain(), 4, D, N) > 0
    assert lib.b2b_chain_vjp_workspace_bytes(chain(n0=5), 4, D, N) == 0
    assert vjp_status(B, chain(n0=5), D) == L_.B2B_EINVAL
    assert vjp_status(B, chain(), D) == L_.B2B_OK
    assert lib.b2b_chain_vjp_workspace_bytes(chain(), 4, 257, N) == 0
    assert vjp_status(B, chain(), 257) == L_.B2B_EUNSUPPORTED


# ---- the Python layer ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("upper,unit", S.FORMS)
def test_python_layer(B, upper, unit):
    import torch

    from bijectors_jl_b200.autograd import _trainable_tensors
    from bijectors_jl_b200.interface import _SLOT_NAMES, _slot_shape, _trainable_slots

    W = getattr(B, S.form_name(upper, unit))
    T = np.arange(16, dtype=np.float32).reshape(4, 4)
    s = B.Scale(W(T), device="cpu")
    assert s.triangular and not s.dense
    assert isinstance(s.a, W) and np.array_equal(s.a.data.numpy(), T)
    assert np.array_equal(s._A.numpy(), T.T)  # column-major storage, as the dense form
    (d,) = s._descs(False, 4)
    assert (d.kind, d.inverse, d.n0, d.n1, d.p0) == (B._lib.SCALE_TRIANGULAR, 0, int(upper), int(unit), s._A.data_ptr())
    (di,) = B.inverse(s)._descs(False, 4)
    assert di.kind == B._lib.SCALE_TRIANGULAR and di.inverse == 1
    assert _SLOT_NAMES[B._lib.SCALE_TRIANGULAR] == ("a",) and _trainable_slots(d) == [0] and _slot_shape(d, 0, 4) == (4, 4)
    assert _trainable_tensors(s)[0] is s._A and _trainable_tensors(B.inverse(s))[0] is s._A
    s64 = B.Scale(W(torch.from_numpy(T)), device="cpu", dtype=torch.float64)
    (d64,) = s64._descs(True, 4, torch.float64)
    assert isinstance(d64, B._lib.LayerDesc64) and d64.kind == B._lib.SCALE_TRIANGULAR and d64.n0 == int(upper)
    with pytest.raises(TypeError):
        s._descs(False, 4, torch.float64)
    with pytest.raises(ValueError, match="DimensionMismatch"):
        s._descs(False, 5)
    with pytest.raises(ValueError, match="DimensionMismatch"):
        W(np.zeros((3, 4)))
    with pytest.raises(ValueError, match="DimensionMismatch"):
        W(torch.zeros(3))
    assert s == B.Scale(W(T.copy()), device="cpu") and s != B.Scale(T, device="cpu")
    with pytest.raises(B.B2BError):
        B.Stacked([s], [(1, 4)], device="cpu")


def test_plain_matrix_is_still_dense(B):
    s = B.Scale(np.eye(3, dtype=np.float32), device="cpu")
    assert s.dense and not s.triangular
    assert s._descs(False, 3)[0].kind == B._lib.SCALE_MATRIX
