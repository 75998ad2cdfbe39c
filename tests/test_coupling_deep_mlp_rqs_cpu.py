"""CPU tests of the deep neural spline coupling reference (tests/coupling_deep_mlp_rqs_oracle.py) and of the host-side
pieces of B2B_COUPLING_DEEP_MLP_RQS: the oracle's reverse mode against central differences, its log-Jacobian against
log|det J| of a finite-difference Jacobian, the inverse, the collapse to the linear spline coupling at LeakyReLU slope 1,
the constructor's errors, the descriptor fields and packed layouts, the constants of the three bindings, and -- with fake
pointers at N = 0, as test_coupling_deep_mlp_cpu.py does it -- the status codes and workspace sizes of the chain entry
points around the envelope."""
import os
import re

import numpy as np
import pytest

import coupling_deep_mlp_rqs_oracle as DR
import spline_coupling_oracle as S

ROOT = os.path.join(os.path.dirname(__file__), "..")
P = 0x10000  # a fake device address: nothing is read through it
ACTS = [("tanh", 0.0), ("leaky_relu", 0.2)]


def _case(rng, n1, n2, H, M, K, scale=0.7):
    """(weights, biases) of an M-hidden-layer network whose last layer gives the (3K − 1)·n1 raw knots."""
    weights = [rng.standard_normal((H, n2)) * scale]
    weights += [rng.standard_normal((H, H)) * scale / np.sqrt(H) for _ in range(M - 1)]
    weights += [rng.standard_normal(((3 * K - 1) * n1, H)) * scale / np.sqrt(H)]
    biases = [rng.standard_normal(H) * 0.5 for _ in range(M)] + [rng.standard_normal((3 * K - 1) * n1) * 0.3]
    return weights, biases


def _fd(f, a, h=1e-6):
    g = np.zeros_like(a)
    for i in np.ndindex(a.shape):
        p, m = a.copy(), a.copy()
        p[i] += h
        m[i] -= h
        g[i] = (f(p) - f(m)) / (2 * h)
    return g


@pytest.mark.parametrize("M", [2, 3, 4])
@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
def test_vjp_matches_central_differences(M, inv, act, slope):
    rng = np.random.default_rng(11 * M + inv + len(act))
    D, N, H, K, B = 6, 3, 4, 3, 2.0
    idx1, idx2 = [2, 5], [6, 3, 1]  # row 4 is an x₃ row
    weights, biases = _case(rng, 2, 3, H, M, K)
    x = rng.standard_normal((D, N)) * 0.8
    x[1, 0] = 3.0  # one element outside the box: the identity
    yb, lb = rng.standard_normal((D, N)), rng.standard_normal(N)
    f = DR.inverse if inv else DR.forward

    def loss(x_, Ws, bs):
        y, lj = f(idx1, idx2, Ws, bs, K, B, act, slope, x_)
        return float(np.sum(y * yb) + np.sum(lj * lb))

    xb, g = DR.vjp(idx1, idx2, weights, biases, K, B, act, slope, x, yb, lb, inverse=inv)

    def check(got, want):
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max())

    check(xb, _fd(lambda a: loss(a, weights, biases), x))
    check(g["W_in"], _fd(lambda a: loss(x, [a] + weights[1:], biases), weights[0]))
    for l in range(1, M):
        check(g["W_hid"][l - 1], _fd(lambda a: loss(x, weights[:l] + [a] + weights[l + 1:], biases), weights[l]))
    check(g["W_out"], _fd(lambda a: loss(x, weights[:-1] + [a], biases), weights[-1]))
    sizes = np.cumsum([len(b) for b in biases])[:-1]
    check(g["c"], _fd(lambda a: loss(x, weights, np.split(a, sizes)), np.concatenate(biases)))


@pytest.mark.parametrize("act,slope", ACTS)
def test_logjac_is_log_det_of_the_jacobian_and_inverse_undoes_forward(act, slope):
    rng = np.random.default_rng(4)
    D, H, K, B = 5, 3, 4, 3.0
    idx1, idx2 = [1, 4], [2, 5]
    weights, biases = _case(rng, 2, 2, H, 3, K)
    x = rng.standard_normal(D)
    for f in (DR.forward, DR.inverse):
        def col(v):
            return f(idx1, idx2, weights, biases, K, B, act, slope, v[:, None])[0][:, 0]

        Jm = np.stack([(col(x + h) - col(x - h)) / 2e-6 for h in np.eye(D) * 1e-6], axis=1)
        lj = f(idx1, idx2, weights, biases, K, B, act, slope, x[:, None])[1][0]
        assert abs(np.log(abs(np.linalg.det(Jm))) - lj) < 1e-6
    X = rng.standard_normal((D, 40)) * 1.5
    for bs in (biases, None):
        y, lj = DR.forward(idx1, idx2, weights, bs, K, B, act, slope, X)
        xr, ljr = DR.inverse(idx1, idx2, weights, bs, K, B, act, slope, y)
        np.testing.assert_allclose(xr, X, atol=1e-10, rtol=0)
        np.testing.assert_allclose(ljr, -lj, atol=1e-10, rtol=0)
        assert np.array_equal(y[[1, 2, 4]], X[[1, 2, 4]])


@pytest.mark.parametrize("M", [2, 3, 4])
def test_slope_one_is_the_linear_spline_coupling_and_tanh_is_not(M):
    """LeakyReLU(1) is the identity, so the layer is the kind-11 spline coupling on W = W_out·W_M⋯W_2·W_in with the
    biases folded: c = W_out·(W_M·(⋯(W_2·c_1 + c_2)⋯) + c_M) + c_out."""
    rng = np.random.default_rng(8 + M)
    D, N, H, K, B = 6, 9, 4, 3, 2.5
    idx1, idx2 = [1, 3], [2, 6, 5]
    weights, biases = _case(rng, 2, 3, H, M, K)
    W, c = weights[0], biases[0]
    for Wl, cl in zip(weights[1:], biases[1:]):
        W, c = Wl @ W, Wl @ c + cl
    x = rng.standard_normal((D, N))
    for fl, fs in ((DR.forward, S.forward), (DR.inverse, S.inverse)):
        ya, la = fs(idx1, idx2, W, c, K, B, x)
        y, lj = fl(idx1, idx2, weights, biases, K, B, "leaky_relu", 1.0, x)
        np.testing.assert_allclose(y, ya, atol=1e-12, rtol=0)
        np.testing.assert_allclose(lj, la, atol=1e-12, rtol=0)
    yt, lt = DR.forward(idx1, idx2, weights, biases, K, B, "tanh", 0.0, x)
    ya, la = S.forward(idx1, idx2, W, c, K, B, x)
    assert np.abs(yt - ya).max() > 1e-3 and np.abs(lt - la).max() > 1e-3


def test_conditioner_errors():
    import torch

    import bijectors_jl_b200 as B

    H, n1, n2, K = 5, 3, 2, 4
    J = (3 * K - 1) * n1
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    Ws = [z(H, n2), z(H, H), z(J, H)]
    bs = [z(H), z(H), z(J)]
    B.DeepMLPSplineConditioner(Ws, bs, K=K, B=3.0, device="cpu")
    with pytest.raises(ValueError, match="MLPSplineConditioner"):
        B.DeepMLPSplineConditioner([z(H, n2), z(J, H)], K=K, B=3.0, device="cpu")  # one hidden layer is kind 14
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner([z(H, n2), z(H, H + 1), z(J, H)], K=K, B=3.0, device="cpu")  # W_2 not H x H
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner([z(H, n2), z(H, H), z(J + 1, H)], K=K, B=3.0, device="cpu")  # rows not (3K−1)·n1
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner([z(H, n2), z(H, H), z(J, H + 1)], K=K, B=3.0, device="cpu")  # columns not H
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner([z(0, n2), z(0, 0), z(J, 0)], K=K, B=3.0, device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner(Ws, K=0, B=3.0, device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner(Ws, K=K, B=0.0, device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner(Ws, bs[:-1], K=K, B=3.0, device="cpu")  # all M + 1 biases or none
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner(Ws, [z(H), z(H + 1), z(J)], K=K, B=3.0, device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner(Ws, [z(H), z(H), z(J - 1)], K=K, B=3.0, device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPSplineConditioner(Ws, K=K, B=3.0, activation="gelu", device="cpu")
    with pytest.raises(TypeError):
        B.DeepMLPSplineConditioner(Ws, K=K, B=3.0, device="cpu", dtype=torch.float64)


@pytest.mark.parametrize("M", [2, 4])
def test_descriptor_and_packed_layouts(M):
    import torch

    import bijectors_jl_b200 as B
    from bijectors_jl_b200 import _lib

    H, n1, n2, K = 5, 3, 2, 3
    J = (3 * K - 1) * n1
    rng = np.random.default_rng(M)
    Ws = [rng.standard_normal(s).astype(np.float32) for s in [(H, n2)] + [(H, H)] * (M - 1) + [(J, H)]]
    bs = [rng.standard_normal(n).astype(np.float32) for n in [H] * M + [J]]
    cond = B.DeepMLPSplineConditioner(Ws, bs, K=K, B=2.5, activation="leaky_relu", slope=0.25, device="cpu")
    assert (cond.n1, cond.n2, cond.H, cond.M, cond.K, cond.B) == (n1, n2, H, M, K, 2.5)
    # W_in / W_out column-major; W_hid [l − 2] = W_l column-major, back to back; c = [c_1 | … | c_M | c_out]
    assert np.array_equal(cond.W_in.numpy().reshape(-1), Ws[0].T.reshape(-1))
    assert np.array_equal(cond.W_out.numpy().reshape(-1), Ws[-1].T.reshape(-1))
    assert tuple(cond.W_hid.shape) == (M - 1, H, H) and cond.W_hid.is_contiguous()
    assert np.array_equal(cond.W_hid.numpy().reshape(-1), np.concatenate([W.T.reshape(-1) for W in Ws[1:-1]]))
    assert np.array_equal(cond.c.numpy(), np.concatenate(bs))
    assert all(np.array_equal(a.numpy(), b) for a, b in zip(cond.weights, Ws)) and len(cond.weights) == M + 1
    assert all(np.array_equal(a.numpy(), b) for a, b in zip(cond.biases, bs)) and len(cond.biases) == M + 1

    mask = B.PartitionMask(7, [2, 4, 6], [1, 7])
    with pytest.raises(ValueError):
        B.Coupling(cond, B.PartitionMask(7, [2, 4], [1, 7]))
    cl = B.Coupling(cond, mask)
    d = cl._descs(True, 7)[0]
    assert (d.kind, d.inverse, d.n0, d.n1, d.n2) == (_lib.COUPLING_DEEP_MLP_RQS, 1, n1, n2, H)
    assert d.n3 == _lib.ACT_LEAKY_RELU | (K << 8) | (M << 16) and (d.f0, d.f1) == (0.25, 2.5)
    assert (d.p0, d.p1, d.p2, d.p3) == tuple(t.data_ptr() for t in (cond.W_in, cond.W_hid, cond.W_out, cond.c))
    assert d.i0 == cl._idx1.data_ptr() and d.i1 == cl._idx2.data_ptr()
    with pytest.raises(TypeError):
        cl._descs(False, 7, torch.float64)

    bare = B.DeepMLPSplineConditioner(Ws, K=K, B=2.5, device="cpu")
    assert bare.c is None and bare.biases is None
    nd = B.Coupling(bare, mask)._descs(False, 7)[0]
    assert nd.p3 is None and nd.n3 == _lib.ACT_TANH | (K << 8) | (M << 16) and nd.f0 == 0.0
    assert B.coupling(cl) is cond and cl == B.Coupling(cond.to("cpu"), mask) and cl != B.Coupling(bare, mask)
    new = lambda **kw: B.Coupling(B.DeepMLPSplineConditioner(Ws, bs, **{**dict(  # noqa: E731
        K=K, B=2.5, activation="leaky_relu", slope=0.25, device="cpu"), **kw}), mask)
    assert cl == new()
    assert cl != new(slope=0.5) and cl != new(activation="tanh") and cl != new(B=2.0)
    Ws2 = Ws[:-1] + [rng.standard_normal(((3 * (K + 1) - 1) * n1, H)).astype(np.float32)]
    assert B.Coupling(bare, mask) != B.Coupling(B.DeepMLPSplineConditioner(Ws2, K=K + 1, B=2.5, device="cpu"), mask)
    deeper = B.DeepMLPSplineConditioner(Ws[:1] + Ws[1:2] * M + Ws[-1:], K=K, B=2.5, device="cpu")
    assert B.Coupling(bare, mask) != B.Coupling(deeper, mask)
    # the affine deep conditioner with the same tensors is a different law
    aff = B.DeepMLPConditioner(Ws[:-1] + [np.zeros((2 * n1, H), np.float32)], device="cpu")
    assert B.Coupling(aff, mask) != B.Coupling(bare, mask)
    assert [t.data_ptr() for t in B.autograd._trainable_tensors(B.Coupling(bare, mask))] == \
        [bare.W_in.data_ptr(), bare.W_hid.data_ptr(), bare.W_out.data_ptr()]
    assert len(B.autograd._trainable_tensors(cl)) == 4
    moved = cond.to("cpu")
    assert (moved.M, moved.K, moved.B) == (M, K, 2.5)
    assert all(torch.equal(a, b) for a, b in zip(moved._tensors(), cond._tensors()))


def test_header_python_and_julia_constants_agree():
    from bijectors_jl_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    jl = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()

    def define(name):
        return int(re.search(rf"#define B2B_{name} (\d+)", hdr).group(1))

    assert define("COUPLING_DEEP_MLP_RQS") == _lib.COUPLING_DEEP_MLP_RQS == 16
    assert "const COUPLING_DEEP_MLP_RQS = Int32(16)" in jl
    assert tuple(define(f"COUPLING_DEEP_MLP_RQS_MAX_{s}") for s in ("N", "H", "K", "DEPTH", "D")) == \
        (_lib.COUPLING_DEEP_MLP_RQS_MAX_N, _lib.COUPLING_DEEP_MLP_RQS_MAX_H, _lib.COUPLING_DEEP_MLP_RQS_MAX_K,
         _lib.COUPLING_DEEP_MLP_RQS_MAX_DEPTH, _lib.COUPLING_DEEP_MLP_RQS_MAX_D) == (128, 128, 16, 4, 1024)
    kinds = {int(v) for v in re.findall(r"#define B2B_[A-Z_]+ (\d+) +/\* [A-Z]", hdr)}
    assert 16 in kinds and 10 not in kinds


# ---- the chain entry points on the host --------------------------------------------------------------------------------
def _deep(n1, n2, H, M, K, act=0, inv=0, c=True, B=3.0, **over):
    from bijectors_jl_b200 import _lib

    d = dict(kind=_lib.COUPLING_DEEP_MLP_RQS, inverse=inv, p0=P, p1=P, p2=P, i0=P, i1=P, n0=n1, n1=n2, n2=H,
             n3=(act & 255) | (K << 8) | (M << 16), f0=0.1, f1=B)
    if c:
        d.update(p3=P)
    d.update(over)
    return d


def _arr(chain, cls):
    a = (cls * len(chain))()
    for d, spec in zip(a, chain):
        for k, v in spec.items():
            setattr(d, k, v)
    return a


def _status(chain, D):
    """(b2b_chain_vjp_f32 status at N = 0 without cotangent pointers, forward workspace, VJP workspace at N = 2²⁰)."""
    from bijectors_jl_b200 import _lib

    L_ = _lib.lib()
    a = _arr(chain, _lib.LayerDesc)
    st = L_.b2b_chain_vjp_f32(a, len(chain), None, None, None, None, None, D, 0, D, D, D, None, 0, None)
    return st, L_.b2b_chain_workspace_bytes(a, len(chain), D, 1 << 20, 1, 0), L_.b2b_chain_vjp_workspace_bytes(a, len(chain), D, 1 << 20)


@pytest.mark.parametrize("n1,n2,H,M,K,D", [(1, 1, 1, 2, 2, 3), (3, 5, 7, 3, 5, 10), (128, 128, 128, 4, 16, 256),
                                           (128, 128, 128, 4, 16, 1024), (64, 128, 32, 2, 8, 1024)])
def test_inside_the_envelope(n1, n2, H, M, K, D):
    for act in (0, 1):
        for inv in (0, 1):
            for c in (True, False):
                st, fwd, vjp = _status([_deep(n1, n2, H, M, K, act, inv, c)], D)
                assert st == 0 and fwd == 0  # the forward launch needs no workspace
                # two D x N cotangent buffers, plus the slices of the parameter sums: those stay under 256 MiB
                assert 0 < vjp - 2 * D * (1 << 20) * 4 <= (256 << 20) + 4096


def test_workspace_grows_with_depth():
    """The per-CTA slice holds W̄_out, c̄_out, W̄_in, c̄_1 and every W̄_l, c̄_l: one more hidden layer adds H² + H floats."""
    sizes = [_status([_deep(8, 8, 32, M, 4)], 64)[2] for M in (2, 3, 4)]
    assert sizes[0] < sizes[1] < sizes[2]


@pytest.mark.parametrize("n1,n2,H,M,K,D", [(129, 1, 4, 2, 4, 300), (1, 129, 4, 2, 4, 300), (4, 4, 129, 2, 4, 40),
                                           (4, 4, 4, 5, 4, 40), (4, 4, 4, 2, 17, 40), (4, 4, 4, 2, 1, 40),
                                           (4, 4, 4, 2, 4, 1025)])
def test_just_past_the_envelope(n1, n2, H, M, K, D):
    assert _status([_deep(n1, n2, H, M, K)], D) == (-2, 0, 0)


def test_invalid_descriptors():
    assert _status([_deep(4, 4, 8, 0, 4)], 16)[0] == -1
    assert _status([_deep(4, 4, 8, 1, 4)], 16)[0] == -1  # one hidden layer is B2B_COUPLING_MLP_RQS
    assert _status([_deep(4, 4, 8, 2, 0)], 16)[0] == -1  # K < 1
    assert _status([_deep(4, 4, 8, 2, 4, B=0.0)], 16)[0] == -1
    assert _status([_deep(4, 4, 8, 2, 4, B=-1.0)], 16)[0] == -1
    assert _status([_deep(4, 4, 8, 2, 4, act=2)], 16)[0] == -1
    assert _status([_deep(4, 4, 8, 2, 4, n3=-1)], 16)[0] == -1
    assert _status([_deep(4, 4, 0, 2, 4)], 16)[0] == -1
    assert _status([_deep(0, 4, 8, 2, 4)], 16)[0] == -1
    assert _status([_deep(4, 0, 8, 2, 4)], 16)[0] == -1
    assert _status([_deep(9, 8, 8, 2, 4)], 16)[0] == -1  # n1 + n2 > D
    for missing in ("p0", "p1", "p2", "i0", "i1"):
        assert _status([_deep(4, 4, 8, 2, 4, **{missing: None})], 16)[0] == -1, missing
    assert _status([_deep(4, 4, 8, 2, 4, c=False)], 16)[0] == 0  # c is optional


def test_float64_entry_points_refuse_the_kind():
    from bijectors_jl_b200 import _lib

    a = _arr([_deep(4, 4, 8, 3, 4)], _lib.LayerDesc64)
    L_ = _lib.lib()
    assert L_.b2b_chain_vjp_workspace_bytes_f64(a, 1, 16, 1000) == 0
    assert L_.b2b_chain_vjp_f64(a, 1, None, None, None, None, None, 16, 0, 16, 16, 16, None, 0, None) == -2


def test_cotangent_slots():
    """A c̄ request needs biases (B2B_EINVAL without); every slot has the shape of its parameter."""
    import ctypes

    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200 import interface as I

    L_ = _lib.lib()
    a = _arr([_deep(4, 4, 8, 3, 5, c=False)], _lib.LayerDesc)
    bars = (ctypes.c_void_p * 4)(None, None, None, P)
    assert L_.b2b_chain_vjp_f32(a, 1, None, None, None, None, bars, 16, 0, 16, 16, 16, None, 0, None) == -1
    d = _arr([_deep(4, 3, 8, 3, 5)], _lib.LayerDesc)[0]
    assert [I._slot_shape(d, i, 16) for i in range(4)] == [(3, 8), (2, 8, 8), (8, 14 * 4), (3 * 8 + 14 * 4,)]


def test_mixed_chain_plans():
    """With planar, BatchNorm, Permute, kind-14 and kind-15 neighbours and a terminal MvNormal: accepted, no forward
    workspace, and the VJP workspace holds one checkpoint per extra segment."""
    from bijectors_jl_b200 import _lib

    D, N = 64, 1 << 20
    planar = dict(kind=_lib.PLANAR, p0=P, p1=P, p2=P)
    bn = dict(kind=_lib.BATCHNORM, p0=P, p1=P, p2=P, p3=P, f0=1e-5)
    perm = dict(kind=_lib.PERMUTE, i0=P)
    diag = dict(kind=_lib.MVNORMAL_DIAG, p0=P, p1=P)
    nsf = dict(kind=_lib.COUPLING_MLP_RQS, p0=P, p1=P, p2=P, p3=P, i0=P, i1=P, n0=32, n1=32, n2=64, n3=8 << 8, f1=3.0)
    dmlp = dict(kind=_lib.COUPLING_DEEP_MLP, p0=P, p1=P, p2=P, p3=P, i0=P, i1=P, n0=32, n1=32, n2=64, n3=2 << 8)
    deep = _deep(32, 32, 64, 3, 8)
    chain = [planar, bn, deep, bn, perm, nsf, dmlp, _deep(32, 32, 64, 2, 4, act=1, inv=1), diag]
    st, fwd, vjp = _status(chain, D)
    assert st == 0 and fwd == 0
    L_ = _lib.lib()
    a = _arr(chain, _lib.LayerDesc)
    assert L_.b2b_chain_workspace_bytes(a, len(chain), D, N, 0, 0) >= D * N * 4
    assert vjp > _status([deep], D)[2] + 4 * D * N * 4
