"""CPU tests of the LU linear layer, B2B_SCALE_LU: the float64 oracle against central differences, the constants of the
header, the Python binding and the Julia shim, the status codes and workspace sizes of the host paths (N = 0 calls and
workspace queries), and the Python layer.  No GPU needed."""
import ctypes
import os
import re

import numpy as np
import pytest

import scale_lu_oracle as S

ROOT = os.path.join(os.path.dirname(__file__), "..")


@pytest.fixture(scope="module")
def B():
    import bijectors_jl_b200 as B

    return B


# ---- the oracle -------------------------------------------------------------------------------------------------------
def _loss(F, dst, x, yb, lb, inv):
    y, lj = (S.inverse if inv else S.forward)(F, dst, x)
    return float(np.sum(yb * y) + np.sum(lb * lj))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("permuted", [False, True])
def test_vjp_matches_central_differences(permuted, inv):
    rng = np.random.default_rng(2 * permuted + inv)
    D, N, h = 5, 4, 1e-6
    F = S.random_lu(rng, D, np.float64)
    dst = rng.permutation(D) if permuted else None
    x, yb, lb = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    xb, Fb = S.vjp(F, dst, x, yb, lb, inverse=inv)
    for i in range(D):
        for n in range(N):
            e = np.zeros_like(x)
            e[i, n] = h
            fd = (_loss(F, dst, x + e, yb, lb, inv) - _loss(F, dst, x - e, yb, lb, inv)) / (2 * h)
            assert abs(fd - xb[i, n]) <= 1e-6 * max(1.0, abs(fd)), (i, n)
    for i in range(D):
        for j in range(D):
            E = np.zeros_like(F)
            E[i, j] = h
            fd = (_loss(F + E, dst, x, yb, lb, inv) - _loss(F - E, dst, x, yb, lb, inv)) / (2 * h)
            assert abs(fd - Fb[i, j]) <= 1e-6 * max(1.0, abs(fd)), (i, j)
    # the log-Jacobian's share: with ȳ = 0, F̄ is ±s·diag(1/Uᵢᵢ) and 0 off the diagonal (∂log|det A|/∂A = A⁻ᵀ through A = PLU)
    _, Fl = S.vjp(F, dst, x, None, lb, inverse=inv)
    want = (-1 if inv else 1) * lb.sum() * np.diag(1.0 / np.diag(F))
    assert np.allclose(Fl, want, rtol=1e-12, atol=1e-12)


def test_oracle_matches_dense_algebra():
    rng = np.random.default_rng(9)
    D = 7
    F = S.random_lu(rng, D, np.float64)
    dst = rng.permutation(D)
    A = S.matrix(F, dst)
    x = rng.standard_normal((D, 3))
    y, lj = S.forward(F, dst, x)
    assert np.allclose(y, A @ x) and np.allclose(lj, np.linalg.slogdet(A)[1])
    xr, lji = S.inverse(F, dst, y)
    assert np.allclose(xr, x) and np.allclose(lji, -lj)
    # y[dst[r]] = (L U x)[r]
    L, U = S.factors(F)
    assert np.allclose(y[dst], L @ U @ x)
    assert np.linalg.cond(A) < 30


# ---- constants ----------------------------------------------------------------------------------------------------------
def test_constants_agree(B):
    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    jl = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()
    assert int(re.search(r"#define B2B_SCALE_LU (\d+)", hdr).group(1)) == B._lib.SCALE_LU == 19
    assert int(re.search(r"#define B2B_SCALE_LU_MAX_D (\d+)", hdr).group(1)) == B._lib.SCALE_LU_MAX_D == 256
    assert int(re.search(r"const SCALE_LU = Int32\((\d+)\)", jl).group(1)) == 19
    assert int(re.search(r"const SCALE_LU_MAX_D = (\d+)", jl).group(1)) == 256
    kinds = [int(v) for v in re.findall(r"#define B2B_[A-Z_]+ (\d+)\s+/\*", hdr)]
    assert 19 in kinds and 10 not in kinds  # 10 stays an invalid kind


# ---- status codes and workspace sizes through the host paths -------------------------------------------------------------
def descs(B, inverse=0, p0=0x1000, i0=None, f64=False, extra=()):
    d = (B._lib.LayerDesc64 if f64 else B._lib.LayerDesc)()
    d.kind, d.inverse, d.p0 = B._lib.SCALE_LU, inverse, p0
    if i0 is not None:
        d.i0 = i0
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
        for i0 in (None, 0x5000):
            assert vjp_status(B, descs(B, i0=i0, f64=f64), 8, f64=f64) == L_.B2B_OK  # N = 0
        assert vjp_status(B, descs(B, p0=None, f64=f64), 8, f64=f64) == L_.B2B_EINVAL
        for slot in (1, 2, 3):
            bars = [None] * 4
            bars[slot] = 0x4000
            assert vjp_status(B, descs(B, f64=f64), 8, bars, f64=f64) == L_.B2B_EUNSUPPORTED, slot
    # the Float32 envelope: D <= 256, refused past it with workspace 0
    for inv in (0, 1):
        a = descs(B, inverse=inv)
        assert vjp_status(B, a, 257) == L_.B2B_EUNSUPPORTED
        assert lib.b2b_chain_workspace_bytes(a, 1, 257, 1000, 1, 0) == 0 and lib.b2b_workspace_bytes(a, 257, 1000) == 0
        assert lib.b2b_chain_vjp_workspace_bytes(a, 1, 257, 1000) == 0
        assert lib.b2b_chain_workspace_bytes(descs(B, inverse=inv), 1, 256, 1000, 1, 0) > 0
    # Float64: D <= 2048
    assert vjp_status(B, descs(B, f64=True), 2048, f64=True) == L_.B2B_OK
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, f64=True), 1, 2048, 100) > 0
    assert vjp_status(B, descs(B, f64=True), 2049, f64=True) == L_.B2B_EUNSUPPORTED
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, f64=True), 1, 2049, 100) == 0
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, p0=None, f64=True), 1, 8, 100) == 0


def test_workspace_formulas(B):
    """The chain workspace holds [M (4·D² B)][log|det U| (8 B)], each rounded up to 256, + 256, as the triangular layer's;
    a chain holding other Scale kinds one region of the largest; the reverse mode adds P·D² floats and 2·D² + 1 doubles,
    P the column chunks of G; the Float64 reverse mode D² doubles of F̄ per warp slot."""
    lib, L_ = B.lib(), B._lib
    for D in (1, 5, 64, 200, 256):
        lu = al256(4 * D * D) + al256(8) + 256
        dense = al256(8 * D * D) + al256(4 * D * D) + al256(4 * D) + al256(8) + 256
        for inv in (0, 1):
            assert lib.b2b_chain_workspace_bytes(descs(B, inverse=inv), 1, D, 1000, 1, 0) == lu
            assert lib.b2b_workspace_bytes(descs(B, inverse=inv), D, 1000) == lu
        dm, dt = L_.LayerDesc(), L_.LayerDesc()
        dm.kind, dm.p0 = L_.SCALE_MATRIX, 0x1000
        dt.kind, dt.p0, dt.n0 = L_.SCALE_TRIANGULAR, 0x1000, 1
        assert lib.b2b_chain_workspace_bytes(descs(B, extra=(dm,)), 2, D, 1000, 1, 0) == dense
        assert lib.b2b_chain_workspace_bytes(descs(B, extra=(dt,)), 2, D, 1000, 1, 0) == lu
        assert lib.b2b_chain_workspace_bytes(descs(B, extra=(dt, dm)), 3, D, 1000, 1, 0) == dense
        for N, P in ((1, 1), (4096, 1), (5000, 2), (1 << 20, 64)):
            want = lu + al256(4 * P * D * D) + 2 * al256(8 * D * D) + al256(8)
            got = lib.b2b_chain_vjp_workspace_bytes(descs(B), 1, D, N)
            # + the chain reverse mode's two D x N cotangent buffers and its alignment slack
            assert got == want + 2 * al256(4 * D * N) + 256, (D, N, got, want)
    # Float64 reverse mode: W warp slots of 8·(T + P) bytes plus 8·P, T = D rounded up to 32, P = D² rounded up to 32
    D, N = 40, 8
    T, P = (D + 31) & ~31, (D * D + 31) & ~31
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, f64=True), 1, D, N) == 8 * 8 * (T + P) + 8 * P + 256


def test_mixed_chains_size_and_refuse_together(B):
    """Inside chains with planar, coupling and MvNormal layers the queries are 0 exactly when a layer is refused."""
    lib, L_ = B.lib(), B._lib
    D, N = 64, 5000

    def chain(p0=0x1400):
        pl, cp, mv = L_.LayerDesc(), L_.LayerDesc(), L_.LayerDesc()
        pl.kind, pl.p0, pl.p1, pl.p2 = L_.PLANAR, 0x1000, 0x1100, 0x1200
        cp.kind, cp.n0, cp.n1, cp.n2, cp.n3, cp.p0 = L_.COUPLING_AFFINE, 32, 32, 0, 32, 0x1300
        mv.kind = L_.MVNORMAL_DIAG
        t = descs(B, p0=p0, i0=0x1500)[0]
        return (L_.LayerDesc * 4)(pl, t, cp, mv)

    assert lib.b2b_chain_workspace_bytes(chain(), 4, D, N, 1, 0) > 0
    assert lib.b2b_chain_vjp_workspace_bytes(chain(), 4, D, N) > 0
    assert lib.b2b_chain_vjp_workspace_bytes(chain(p0=None), 4, D, N) == 0
    assert vjp_status(B, chain(p0=None), D) == L_.B2B_EINVAL
    assert vjp_status(B, chain(), D) == L_.B2B_OK
    assert lib.b2b_chain_vjp_workspace_bytes(chain(), 4, 257, N) == 0
    assert vjp_status(B, chain(), 257) == L_.B2B_EUNSUPPORTED


# ---- the Python layer ---------------------------------------------------------------------------------------------------
def test_python_layer(B):
    import torch

    from bijectors_jl_b200.autograd import _trainable_tensors
    from bijectors_jl_b200.interface import _SLOT_NAMES, _slot_shape, _trainable_slots

    F = np.arange(16, dtype=np.float32).reshape(4, 4) + 1
    p = [3, 1, 4, 2]
    lay = B.LULinear(F, p, device="cpu")
    assert np.array_equal(lay._F.numpy(), F.T)  # column-major storage, as a dense Scale
    assert np.array_equal(lay.factors.numpy(), F) and np.array_equal(lay.p, p)
    assert isinstance(lay.L, B.UnitLowerTriangular) and isinstance(lay.U, B.UpperTriangular)
    assert np.array_equal(lay.L.data.numpy(), F) and np.array_equal(lay.U.data.numpy(), F)
    (d,) = lay._descs(False, 4)
    assert (d.kind, d.inverse, d.p0, d.i0) == (B._lib.SCALE_LU, 0, lay._F.data_ptr(), lay._dst.data_ptr())
    assert lay._dst.tolist() == [2, 0, 3, 1]  # 0-based destination rows
    (di,) = B.inverse(lay)._descs(False, 4)
    assert di.kind == B._lib.SCALE_LU and di.inverse == 1
    (dn,) = B.LULinear(F, device="cpu")._descs(False, 4)
    assert not dn.i0 and np.array_equal(B.LULinear(F, device="cpu").p, [1, 2, 3, 4])
    assert _SLOT_NAMES[B._lib.SCALE_LU] == ("factors",) and _trainable_slots(d) == [0] and _slot_shape(d, 0, 4) == (4, 4)
    assert _trainable_tensors(lay) == [lay._F] and _trainable_tensors(B.inverse(lay))[0] is lay._F
    l64 = B.LULinear(torch.from_numpy(F), p, device="cpu", dtype=torch.float64)
    (d64,) = l64._descs(True, 4, torch.float64)
    assert isinstance(d64, B._lib.LayerDesc64) and d64.kind == B._lib.SCALE_LU and d64.i0 == l64._dst.data_ptr()
    with pytest.raises(TypeError):
        lay._descs(False, 4, torch.float64)
    with pytest.raises(ValueError, match="DimensionMismatch"):
        lay._descs(False, 5)
    with pytest.raises(ValueError, match="DimensionMismatch"):
        B.LULinear(np.zeros((3, 4)), device="cpu")
    with pytest.raises(ValueError, match="DimensionMismatch"):
        B.LULinear(np.zeros(3), device="cpu")
    with pytest.raises(ValueError, match="DimensionMismatch"):
        B.LULinear(F, [1, 2, 3], device="cpu")
    for bad in ([1, 1, 2, 3], [0, 1, 2, 3], [1, 2, 3, 5]):
        with pytest.raises(ValueError, match="permutation"):
            B.LULinear(F, bad, device="cpu")
    assert lay == B.LULinear(F.copy(), list(p), device="cpu")
    assert lay != B.LULinear(F, device="cpu") and lay != B.LULinear(F + 1, p, device="cpu")
    assert B.LULinear(F, device="cpu") == B.LULinear(F, [1, 2, 3, 4], device="cpu")
    moved = lay.to("cpu")
    assert moved == lay and moved._dst is not None


def test_from_matrix_gives_back_the_matrix(B):
    rng = np.random.default_rng(5)
    for D in (1, 2, 7, 64):
        A = rng.standard_normal((D, D))
        lay = B.LULinear.from_matrix(A, device="cpu", dtype=__import__("torch").float64)
        F = lay.factors.numpy()
        assert np.allclose(S.matrix(F, lay.p - 1), A, rtol=1e-12, atol=1e-12)
        L, _ = S.factors(F)
        assert np.abs(np.tril(L, -1)).max(initial=0.0) <= 1.0  # partial pivoting: |Lᵢⱼ| <= 1
        l32 = B.LULinear.from_matrix(A, device="cpu")
        assert np.allclose(S.matrix(l32.factors.numpy(), l32.p - 1), A, rtol=1e-5, atol=1e-5)
