"""CPU tests of the masked autoregressive layer, B2B_AUTOREGRESSIVE_MLP: the float64 oracle (triangular Jacobian,
log-determinant, inverse, both reverse rules against central differences), the constants of the header, the Python
binding and the Julia shim, the status codes and workspace queries of the entry points with nothing launched, and the
Python layer.  No GPU needed."""
import ctypes
import os
import re

import numpy as np
import pytest

import autoregressive_oracle as A

ROOT = os.path.join(os.path.dirname(__file__), "..")
ACTS = [("tanh", 0.0), ("leaky_relu", 0.3)]


@pytest.fixture(scope="module")
def B():
    import bijectors_jl_b200 as B

    return B


def params(rng, D, H, deg="random", with_c=True):
    W1, W2 = rng.standard_normal((H, D)) * 0.7, rng.standard_normal((2 * D, H)) * 0.4
    c1 = rng.standard_normal(H) * 0.3 if with_c else None
    c2 = rng.standard_normal(2 * D) * 0.2 if with_c else None
    m = rng.integers(-2, D + 3, H) if deg == "random" else A.default_degrees(D, H)
    return W1, c1, W2, c2, m


def jacobian(f, x, h=1e-6):
    D = x.shape[0]
    J = np.zeros((D, D))
    for r in range(D):
        e = np.zeros((D, 1))
        e[r] = h
        J[:, r] = (f(x + e)[0] - f(x - e)[0])[:, 0] / (2 * h)
    return J


# ---- the oracle -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act,slope", ACTS)
def test_jacobian_is_lower_triangular_with_logdet(act, slope):
    rng = np.random.default_rng(1 if act == "tanh" else 2)
    D, H = 6, 11
    p = params(rng, D, H)
    assert (p[4] <= 0).any() and (p[4] >= D).any()
    x = rng.standard_normal((D, 1))
    J = jacobian(lambda v: A.forward(*p, act, slope, v), x)
    assert np.abs(np.triu(J, 1)).max() == 0.0
    assert np.isclose(np.linalg.slogdet(J)[1], A.forward(*p, act, slope, x)[1][0], rtol=0, atol=1e-7)
    Ji = jacobian(lambda v: A.inverse(*p, act, slope, v), x)
    assert np.abs(np.triu(Ji, 1)).max() == 0.0
    assert np.isclose(np.linalg.slogdet(Ji)[1], A.inverse(*p, act, slope, x)[1][0], rtol=0, atol=1e-7)


@pytest.mark.parametrize("act,slope", ACTS)
def test_inverse_of_forward(act, slope):
    rng = np.random.default_rng(3)
    D, H = 9, 20
    p = params(rng, D, H, deg="default")
    x = rng.standard_normal((D, 13))
    y, lj = A.forward(*p, act, slope, x)
    xr, lji = A.inverse(*p, act, slope, y)
    assert np.allclose(xr, x, rtol=0, atol=1e-10) and np.allclose(lji, -lj, rtol=0, atol=1e-10)


def _loss(p, act, slope, x, yb, lb, inv):
    y, lj = (A.inverse if inv else A.forward)(*p, act, slope, x)
    return float(np.sum(yb * y) + np.sum(lb * lj))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
def test_vjp_matches_central_differences(act, slope, inv):
    rng = np.random.default_rng(4 + inv)
    D, H, N, h = 5, 7, 3, 1e-6
    p = list(params(rng, D, H))
    x, yb, lb = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    xb, g = A.vjp(*p, act, slope, x, yb, lb, inverse=inv)
    for i in range(D):
        for n in range(N):
            e = np.zeros_like(x)
            e[i, n] = h
            fd = (_loss(p, act, slope, x + e, yb, lb, inv) - _loss(p, act, slope, x - e, yb, lb, inv)) / (2 * h)
            assert abs(fd - xb[i, n]) <= 1e-6 * max(1.0, abs(fd)), (i, n)
    M1, M2 = A.masks(p[4], D)
    for slot, name, mask in ((0, "W1", M1), (1, "c1", None), (2, "W2", M2), (3, "c2", None)):
        P = p[slot]
        for idx in np.ndindex(P.shape):
            E = np.zeros_like(P)
            E[idx] = h
            q1, q2 = list(p), list(p)
            q1[slot], q2[slot] = P + E, P - E
            fd = (_loss(q1, act, slope, x, yb, lb, inv) - _loss(q2, act, slope, x, yb, lb, inv)) / (2 * h)
            assert abs(fd - g[name][idx]) <= 1e-6 * max(1.0, abs(fd)), (name, idx)
            if mask is not None and not mask[idx]:
                assert g[name][idx] == 0.0  # exactly 0 outside the masks
    # the log-Jacobian's share alone
    xl, _ = A.vjp(*p, act, slope, x, None, lb, inverse=inv)
    for i in range(D):
        e = np.zeros_like(x)
        e[i] = h
        fd = (_loss(p, act, slope, x + e, 0, lb, inv) - _loss(p, act, slope, x - e, 0, lb, inv)) / (2 * h)
        assert abs(fd - xl[i].sum()) <= 1e-6 * max(1.0, abs(fd))


def test_oracle_as_a_chain_element():
    from oracle import oracle_np as O
    import chain_vjp_oracle as V

    rng = np.random.default_rng(6)
    D, H, N = 4, 6, 5
    lay = A.AutoregressiveLayer(*params(rng, D, H))
    perm = O.Layer("permute", dict(A=O.permute_matrix_from_indices(rng.permutation(D) + 1)))
    x = rng.standard_normal((D, N))
    y, lj = O.chain_forward([lay, perm, lay], x)
    xr, lji = O.chain_inverse([lay, perm, lay], y)
    assert np.allclose(xr, x, atol=1e-12) and np.allclose(lji, -lj, atol=1e-12)
    yb, lb = rng.standard_normal((D, N)), rng.standard_normal(N)
    xb, grads, _ = V.chain_vjp([lay, perm, lay], [True, False, False], x, yb, lb)
    assert xb.shape == (D, N) and set(grads[0]) == {"W1", "c1", "W2", "c2"}


# ---- constants, kind table and status codes --------------------------------------------------------------------------
def test_header_python_and_julia_constants_agree(B):
    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    jl = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()
    L_ = B._lib
    assert int(re.search(r"#define B2B_AUTOREGRESSIVE_MLP (\d+)", hdr).group(1)) == L_.AUTOREGRESSIVE_MLP == 20
    assert int(re.search(r"#define B2B_AUTOREGRESSIVE_MLP_MAX_D (\d+)", hdr).group(1)) == L_.AUTOREGRESSIVE_MLP_MAX_D == 128
    assert int(re.search(r"#define B2B_AUTOREGRESSIVE_MLP_MAX_H (\d+)", hdr).group(1)) == L_.AUTOREGRESSIVE_MLP_MAX_H == 256
    assert int(re.search(r"const AUTOREGRESSIVE_MLP = Int32\((\d+)\)", jl).group(1)) == 20
    assert int(re.search(r"const AUTOREGRESSIVE_MLP_MAX_D = (\d+)", jl).group(1)) == 128
    assert int(re.search(r"const AUTOREGRESSIVE_MLP_MAX_H = (\d+)", jl).group(1)) == 256
    kinds = [int(v) for v in re.findall(r"#define B2B_[A-Z_]+ (\d+)\s+/\*", hdr)]
    assert 20 in kinds and 10 not in kinds  # 10 stays an invalid kind


def desc(B, D=8, H=16, inverse=0, p0=0x1000, p1=0x1100, p2=0x1200, p3=0x1300, i0=0x1400, act=0):
    d = B._lib.LayerDesc()
    d.kind, d.inverse, d.n2, d.n3 = B._lib.AUTOREGRESSIVE_MLP, inverse, H, act
    d.p0, d.p1, d.p2, d.p3, d.i0 = p0, p1, p2, p3, i0
    return (B._lib.LayerDesc * 1)(d)


def run_status(B, arr, D):  # N = 0: nothing is launched
    return B.lib().b2b_chain_run_f32(arr, 1, 0x2000, 0x3000, None, None, D, 0, D, D, 0, None, 0, None)


def vjp_status(B, arr, D, bars=None):
    pb = None
    if bars is not None:
        pb = ctypes.cast((ctypes.c_void_p * 4)(*bars), ctypes.c_void_p)
    return B.lib().b2b_chain_vjp_f32(arr, 1, 0x2000, None, None, 0x3000, pb, D, 0, D, D, D, None, 0, None)


@pytest.mark.parametrize("inverse", [0, 1])
def test_status_codes(B, inverse):
    L_, lib = B._lib, B.lib()
    for kw in (dict(p0=None), dict(p2=None), dict(i0=None), dict(act=2), dict(act=-1), dict(H=0)):
        a = desc(B, inverse=inverse, **kw)
        assert vjp_status(B, a, 8) == L_.B2B_EINVAL, kw
        assert lib.b2b_chain_workspace_bytes(a, 1, 8, 1000, 1, 0) >= 0
    ok = desc(B, inverse=inverse)
    assert vjp_status(B, ok, 8) == L_.B2B_OK  # N = 0
    # a c̄ request without its c
    for slot, kw in ((1, dict(p1=None)), (3, dict(p3=None))):
        bars = [None] * 4
        bars[slot] = 0x4000
        assert vjp_status(B, desc(B, inverse=inverse, **kw), 8, bars) == L_.B2B_EINVAL
        assert run_status(B, desc(B, inverse=inverse, **kw), 8) == L_.B2B_OK
    # the envelope: D <= 128, H <= 256; beyond it refused with workspace 0
    for D, H in ((129, 16), (8, 257), (200, 300)):
        a = desc(B, D=D, H=H, inverse=inverse)
        assert vjp_status(B, a, D) == L_.B2B_EUNSUPPORTED
        assert lib.b2b_chain_workspace_bytes(a, 1, D, 1000, 1, 0) == 0 and lib.b2b_workspace_bytes(a, D, 1000) == 0
        assert lib.b2b_chain_vjp_workspace_bytes(a, 1, D, 1000) == 0
    for D, H in ((1, 1), (128, 256)):
        a = desc(B, D=D, H=H, inverse=inverse)
        hd = D * H * 4
        al = lambda b: (b + 255) & ~255  # noqa: E731
        assert lib.b2b_chain_workspace_bytes(a, 1, D, 1000, 1, 0) == al(hd) + 2 * al(2 * hd) + 256
        assert lib.b2b_chain_vjp_workspace_bytes(a, 1, D, 1000) > 0
        assert vjp_status(B, a, D) == L_.B2B_OK


# ---- the Python layer -------------------------------------------------------------------------------------------------
def test_python_layer(B):
    import torch

    rng = np.random.default_rng(8)
    D, H = 5, 12
    W1, c1, W2, c2, _ = params(rng, D, H)
    lay = B.MaskedAutoregressive(W1, c1, W2, c2, device="cpu")
    m = lay.degrees
    assert m.tolist() == [((k - 1) % (D - 1)) + 1 for k in range(1, H + 1)] == A.default_degrees(D, H).tolist()
    M1, M2 = lay.masks
    O1, O2 = A.masks(m, D)
    assert np.array_equal(M1.cpu().numpy(), O1) and np.array_equal(M2.cpu().numpy(), O2)
    assert torch.equal(lay.W1, torch.as_tensor(W1, dtype=torch.float32)) and lay.W2.shape == (2 * D, H)
    assert lay.c1.shape == (H,) and lay.c2.shape == (2 * D,)
    assert B.MaskedAutoregressive(W1[:, :1], None, W2[:2], None, device="cpu").degrees.tolist() == [1] * H  # D = 1
    assert lay == B.MaskedAutoregressive(W1, c1, W2, c2, device="cpu")
    assert lay != B.MaskedAutoregressive(W1, None, W2, c2, device="cpu")
    assert lay != B.MaskedAutoregressive(W1, c1, W2, c2, degrees=np.ones(H, int), device="cpu")
    assert B.inverse(B.inverse(lay)) is lay and isinstance(B.inverse(lay), B.Inverse)
    d = lay._descs(False, D)[0]
    assert (d.kind, d.inverse, d.n2, d.n3) == (B._lib.AUTOREGRESSIVE_MLP, 0, H, B._lib.ACT_TANH)
    assert d.p0 == lay._W1.data_ptr() and d.p2 == lay._W2.data_ptr() and d.i0 == lay._deg.data_ptr()
    di = B.inverse(B.MaskedAutoregressive(W1, None, W2, None, activation="leaky_relu", slope=0.2, device="cpu"))._descs(False, D)[0]
    assert di.inverse == 1 and not di.p1 and not di.p3 and di.n3 == B._lib.ACT_LEAKY_RELU and abs(di.f0 - 0.2) < 1e-7
    assert set(lay.params()) == {"W1", "c1", "W2", "c2"}
    with pytest.raises(ValueError, match="DimensionMismatch"):
        lay._descs(False, D + 1)
    for bad in (dict(W2=W2[:-1]), dict(W1=W1[:, :-1]), dict(W1=W1[0]), dict(degrees=np.ones(H - 1))):
        kw = dict(W1=W1, c1=c1, W2=W2, c2=c2)
        kw.update(bad)
        with pytest.raises(ValueError, match="DimensionMismatch"):
            B.MaskedAutoregressive(**kw, device="cpu")
    with pytest.raises(ValueError):
        B.MaskedAutoregressive(W1, c1[:-1], W2, c2, device="cpu")
    with pytest.raises(ValueError, match="activation"):
        B.MaskedAutoregressive(W1, c1, W2, c2, activation="relu", device="cpu")
    with pytest.raises(TypeError):
        B.MaskedAutoregressive(W1, c1, W2, c2, device="cpu", dtype=torch.float64)
