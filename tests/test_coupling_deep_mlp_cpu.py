"""CPU tests of the deep neural-network coupling reference (tests/coupling_deep_mlp_oracle.py) and of the host-side pieces
of B2B_COUPLING_DEEP_MLP: the oracle's reverse mode against central differences, its log-Jacobian against log|det J| of a
finite-difference Jacobian, the inverse, the collapse to the affine coupling at LeakyReLU slope 1, the constructor's
errors, the descriptor fields and packed layouts, the constants of the three bindings, and -- with fake pointers at
N = 0, as test_coupling_mlp_cpu.py does it -- the status codes and workspace sizes of the chain entry points around the
envelope."""
import os
import re

import numpy as np
import pytest

import coupling_deep_mlp_oracle as DM
from oracle import oracle_np as O

ROOT = os.path.join(os.path.dirname(__file__), "..")
P = 0x10000  # a fake device address: nothing is read through it


def _case(rng, n1, n2, H, M, scale=0.7):
    """(weights, biases) of an M-hidden-layer network, scaled so that every layer stays in tanh's sensitive range."""
    weights = [rng.standard_normal((H, n2)) * scale]
    weights += [rng.standard_normal((H, H)) * scale / np.sqrt(H) for _ in range(M - 1)]
    weights += [rng.standard_normal((2 * n1, H)) * scale / np.sqrt(H)]
    biases = [rng.standard_normal(H) * 0.5 for _ in range(M)] + [rng.standard_normal(2 * n1) * 0.3]
    return weights, biases


def _fd(f, a, h=1e-6):
    g = np.zeros_like(a)
    for i in np.ndindex(a.shape):
        p, m = a.copy(), a.copy()
        p[i] += h
        m[i] -= h
        g[i] = (f(p) - f(m)) / (2 * h)
    return g


ACTS = [("tanh", 0.0), ("leaky_relu", 0.2), ("leaky_relu", 0.0)]


@pytest.mark.parametrize("M", [2, 3])
@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
def test_vjp_matches_central_differences(M, inv, act, slope):
    rng = np.random.default_rng(int(10 * slope) + inv + len(act) + 7 * M)
    D, N, H = 6, 4, 5
    idx1, idx2 = [2, 5, 1], [6, 3]  # row 4 is an x₃ row
    weights, biases = _case(rng, 3, 2, H, M)
    x = rng.standard_normal((D, N))
    yb, lb = rng.standard_normal((D, N)), rng.standard_normal(N)
    f = DM.inverse if inv else DM.forward

    def loss(x_, Ws, bs):
        y, lj = f(idx1, idx2, Ws, bs, act, slope, x_)
        return float(np.sum(y * yb) + np.sum(lj * lb))

    xb, g = DM.vjp(idx1, idx2, weights, biases, act, slope, x, yb, lb, inverse=inv)

    def check(got, want):
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= 2e-6 * max(1.0, np.abs(want).max())

    check(xb, _fd(lambda a: loss(a, weights, biases), x))
    check(g["W_in"], _fd(lambda a: loss(x, [a] + weights[1:], biases), weights[0]))
    for l in range(1, M):
        check(g["W_hid"][l - 1], _fd(lambda a: loss(x, weights[:l] + [a] + weights[l + 1:], biases), weights[l]))
    check(g["W_out"], _fd(lambda a: loss(x, weights[:-1] + [a], biases), weights[-1]))
    c = np.concatenate(biases)
    sizes = np.cumsum([len(b) for b in biases])[:-1]
    check(g["c"], _fd(lambda a: loss(x, weights, np.split(a, sizes)), c))
    if slope > 0 or act == "tanh":  # with ReLU and c = 0, a column whose h_{l−1} is all zero sits on the kink
        _, g0 = DM.vjp(idx1, idx2, weights, None, act, slope, x, yb, lb, inverse=inv)  # no biases: c̄ at c = 0
        zero = np.zeros_like(c)
        check(g0["c"], _fd(lambda a: loss(x, weights, np.split(a, sizes)), zero))


@pytest.mark.parametrize("act,slope", ACTS)
def test_logjac_is_log_det_of_the_jacobian(act, slope):
    rng = np.random.default_rng(4)
    D, H = 5, 3
    idx1, idx2 = [1, 4], [2, 5]
    weights, biases = _case(rng, 2, 2, H, 3)
    x = rng.standard_normal(D)
    for f in (DM.forward, DM.inverse):
        def col(v):
            return f(idx1, idx2, weights, biases, act, slope, v[:, None])[0][:, 0]

        Jm = np.stack([(col(x + h) - col(x - h)) / 2e-6 for h in np.eye(D) * 1e-6], axis=1)
        lj = f(idx1, idx2, weights, biases, act, slope, x[:, None])[1][0]
        assert abs(np.log(abs(np.linalg.det(Jm))) - lj) < 1e-6


@pytest.mark.parametrize("M", [2, 4])
def test_inverse_of_forward(M):
    rng = np.random.default_rng(6)
    D, N, H = 7, 30, 4
    idx1, idx2 = [7, 1, 3], [2, 4, 6]
    weights, biases = _case(rng, 3, 3, H, M)
    x = rng.standard_normal((D, N))
    for bs in (biases, None):
        y, lj = DM.forward(idx1, idx2, weights, bs, "tanh", 0.0, x)
        xr, ljr = DM.inverse(idx1, idx2, weights, bs, "tanh", 0.0, y)
        np.testing.assert_allclose(xr, x, atol=1e-12, rtol=0)
        np.testing.assert_allclose(ljr, -lj, atol=1e-12, rtol=0)
        assert np.array_equal(y[[1, 3, 4, 5]], x[[1, 3, 4, 5]])


@pytest.mark.parametrize("M", [2, 3, 4])
def test_slope_one_is_the_affine_coupling_and_tanh_is_not(M):
    """LeakyReLU(1) is the identity, so the layer is the affine coupling on W = W_out·W_M⋯W_2·W_in with the biases
    folded: c = W_out·(W_M·(⋯(W_2·c_1 + c_2)⋯) + c_M) + c_out."""
    rng = np.random.default_rng(8 + M)
    D, N, H = 6, 9, 4
    idx1, idx2 = [1, 3], [2, 6, 5]
    weights, biases = _case(rng, 2, 3, H, M)
    W, c = weights[0], biases[0]
    for Wl, cl in zip(weights[1:], biases[1:]):
        W, c = Wl @ W, Wl @ c + cl
    x = rng.standard_normal((D, N))
    ya, la = O.coupling_affine_forward(idx1, idx2, W, c, x)
    y, lj = DM.forward(idx1, idx2, weights, biases, "leaky_relu", 1.0, x)
    np.testing.assert_allclose(y, ya, atol=1e-12, rtol=0)
    np.testing.assert_allclose(lj, la, atol=1e-12, rtol=0)
    yt, lt = DM.forward(idx1, idx2, weights, biases, "tanh", 0.0, x)
    assert np.abs(yt - ya).max() > 1e-2 and np.abs(lt - la).max() > 1e-2


def test_conditioner_errors():
    import torch

    import bijectors_jl_b200 as B

    H, n1, n2 = 5, 3, 2
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    Ws = [z(H, n2), z(H, H), z(2 * n1, H)]
    bs = [z(H), z(H), z(2 * n1)]
    B.DeepMLPConditioner(Ws, bs, device="cpu")
    with pytest.raises(ValueError, match="MLPConditioner"):
        B.DeepMLPConditioner([z(H, n2), z(2 * n1, H)], device="cpu")  # one hidden layer is kind 13
    with pytest.raises(ValueError):
        B.DeepMLPConditioner([z(H, n2), z(H, H + 1), z(2 * n1, H)], device="cpu")  # W_2 not H x H
    with pytest.raises(ValueError):
        B.DeepMLPConditioner([z(H, n2), z(H, H), z(2 * n1 + 1, H)], device="cpu")  # odd row count
    with pytest.raises(ValueError):
        B.DeepMLPConditioner([z(H, n2), z(H, H), z(2 * n1, H + 1)], device="cpu")  # W_out's columns are not H
    with pytest.raises(ValueError):
        B.DeepMLPConditioner([z(0, n2), z(0, 0), z(2 * n1, 0)], device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPConditioner(Ws, bs[:-1], device="cpu")  # all M + 1 biases or none
    with pytest.raises(ValueError):
        B.DeepMLPConditioner(Ws, [z(H), z(H + 1), z(2 * n1)], device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPConditioner(Ws, [z(H), z(H), z(2 * n1 - 1)], device="cpu")
    with pytest.raises(ValueError):
        B.DeepMLPConditioner(Ws, activation="gelu", device="cpu")
    with pytest.raises(TypeError):
        B.DeepMLPConditioner(Ws, device="cpu", dtype=torch.float64)


@pytest.mark.parametrize("M", [2, 4])
def test_descriptor_and_packed_layouts(M):
    import torch

    import bijectors_jl_b200 as B
    from bijectors_jl_b200 import _lib

    H, n1, n2 = 5, 3, 2
    rng = np.random.default_rng(M)
    Ws = [rng.standard_normal(s).astype(np.float32) for s in [(H, n2)] + [(H, H)] * (M - 1) + [(2 * n1, H)]]
    bs = [rng.standard_normal(n).astype(np.float32) for n in [H] * M + [2 * n1]]
    cond = B.DeepMLPConditioner(Ws, bs, activation="leaky_relu", slope=0.25, device="cpu")
    assert (cond.n1, cond.n2, cond.H, cond.M) == (n1, n2, H, M)
    # W_in / W_out column-major; W_hid [l − 2] = W_l column-major, back to back; c = [c_1 | … | c_M | c_out]
    assert np.array_equal(cond.W_in.numpy().reshape(-1), Ws[0].T.reshape(-1))
    assert np.array_equal(cond.W_out.numpy().reshape(-1), Ws[-1].T.reshape(-1))
    assert tuple(cond.W_hid.shape) == (M - 1, H, H) and cond.W_hid.is_contiguous()
    assert np.array_equal(cond.W_hid.numpy().reshape(-1), np.concatenate([W.T.reshape(-1) for W in Ws[1:-1]]))
    assert np.array_equal(cond.c.numpy(), np.concatenate(bs))
    assert all(np.array_equal(a.numpy(), b) for a, b in zip(cond.weights, Ws)) and len(cond.weights) == M + 1
    assert all(np.array_equal(a.numpy(), b) for a, b in zip(cond.biases, bs)) and len(cond.biases) == M + 1
    assert cond.weights[0].data_ptr() == cond.W_in.data_ptr()  # views, not copies
    assert cond.biases[-1].data_ptr() == cond.c.data_ptr() + 4 * M * H

    mask = B.PartitionMask(7, [2, 4, 6], [1, 7])
    with pytest.raises(ValueError):
        B.Coupling(cond, B.PartitionMask(7, [2, 4], [1, 7]))
    cl = B.Coupling(cond, mask)
    d = cl._descs(True, 7)[0]
    assert (d.kind, d.inverse, d.n0, d.n1, d.n2) == (_lib.COUPLING_DEEP_MLP, 1, n1, n2, H) and d.f0 == 0.25
    assert d.n3 == _lib.ACT_LEAKY_RELU | (M << 8)
    assert (d.p0, d.p1, d.p2, d.p3) == tuple(t.data_ptr() for t in (cond.W_in, cond.W_hid, cond.W_out, cond.c))
    assert d.i0 == cl._idx1.data_ptr() and d.i1 == cl._idx2.data_ptr()
    with pytest.raises(TypeError):
        cl._descs(False, 7, torch.float64)

    bare = B.DeepMLPConditioner(Ws, device="cpu")
    assert bare.c is None and bare.biases is None
    nd = B.Coupling(bare, mask)._descs(False, 7)[0]
    assert nd.p3 is None and nd.n3 == _lib.ACT_TANH | (M << 8) and nd.f0 == 0.0
    assert B.coupling(cl) is cond and cl == B.Coupling(cond.to("cpu"), mask) and cl != B.Coupling(bare, mask)
    assert cl != B.Coupling(B.DeepMLPConditioner(Ws, bs, activation="leaky_relu", slope=0.5, device="cpu"), mask)
    assert cl != B.Coupling(B.DeepMLPConditioner(Ws, bs, activation="tanh", device="cpu"), mask)
    deeper = B.DeepMLPConditioner(Ws[:1] + Ws[1:2] * M + Ws[-1:], device="cpu")
    assert B.Coupling(bare, mask) != B.Coupling(deeper, mask)
    assert [t.data_ptr() for t in B.autograd._trainable_tensors(B.Coupling(bare, mask))] == \
        [bare.W_in.data_ptr(), bare.W_hid.data_ptr(), bare.W_out.data_ptr()]
    assert len(B.autograd._trainable_tensors(cl)) == 4
    moved = cond.to("cpu")
    assert moved.M == M and all(torch.equal(a, b) for a, b in zip(moved._tensors(), cond._tensors()))


def test_header_python_and_julia_constants_agree():
    from bijectors_jl_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    jl = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()

    def define(name):
        return int(re.search(rf"#define B2B_{name} (\d+)", hdr).group(1))

    assert define("COUPLING_DEEP_MLP") == _lib.COUPLING_DEEP_MLP == 15 and "const COUPLING_DEEP_MLP = Int32(15)" in jl
    assert tuple(define(f"COUPLING_DEEP_MLP_MAX_{s}") for s in ("N", "H", "DEPTH", "D")) == \
        (_lib.COUPLING_DEEP_MLP_MAX_N, _lib.COUPLING_DEEP_MLP_MAX_H, _lib.COUPLING_DEEP_MLP_MAX_DEPTH,
         _lib.COUPLING_DEEP_MLP_MAX_D) == (128, 128, 4, 1024)
    kinds = {int(v) for v in re.findall(r"#define B2B_[A-Z_]+ (\d+) +/\* [A-Z]", hdr)}
    assert 15 in kinds and 10 not in kinds


# ---- the chain entry points on the host --------------------------------------------------------------------------------
def _deep(n1, n2, H, M, act=0, inv=0, c=True, **over):
    from bijectors_jl_b200 import _lib

    d = dict(kind=_lib.COUPLING_DEEP_MLP, inverse=inv, p0=P, p1=P, p2=P, i0=P, i1=P, n0=n1, n1=n2, n2=H,
             n3=(act & 255) | (M << 8), f0=0.1)
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


@pytest.mark.parametrize("n1,n2,H,M,D", [(1, 1, 1, 2, 3), (3, 5, 7, 3, 10), (128, 128, 128, 4, 256),
                                         (128, 128, 128, 4, 1024)])
def test_inside_the_envelope(n1, n2, H, M, D):
    for act in (0, 1):
        for inv in (0, 1):
            for c in (True, False):
                st, fwd, vjp = _status([_deep(n1, n2, H, M, act, inv, c)], D)
                assert st == 0 and fwd == 0  # the forward launch needs no workspace
                # two D x N cotangent buffers, plus the slices of the parameter sums: those stay under 256 MiB
                assert 0 < vjp - 2 * D * (1 << 20) * 4 <= (256 << 20) + 4096


def test_workspace_grows_with_depth():
    """The per-CTA slice holds W̄_in, every W̄_l, W̄_out and c̄: one more hidden layer adds H² + H floats per slice."""
    sizes = [_status([_deep(64, 64, 128, M)], 128)[2] for M in (2, 3, 4)]
    assert sizes[0] < sizes[1] < sizes[2]


@pytest.mark.parametrize("n1,n2,H,M,D", [(129, 1, 4, 2, 300), (1, 129, 4, 2, 300), (4, 4, 129, 2, 40),
                                         (4, 4, 4, 5, 40), (4, 4, 4, 2, 1025)])
def test_just_past_the_envelope(n1, n2, H, M, D):
    assert _status([_deep(n1, n2, H, M)], D) == (-2, 0, 0)


def test_invalid_descriptors():
    assert _status([_deep(4, 4, 8, 0)], 16)[0] == -1
    assert _status([_deep(4, 4, 8, 1)], 16)[0] == -1  # one hidden layer is B2B_COUPLING_MLP
    assert _status([_deep(4, 4, 8, 2, act=2)], 16)[0] == -1
    assert _status([_deep(4, 4, 8, 2, n3=-1)], 16)[0] == -1
    assert _status([_deep(4, 4, 0, 2)], 16)[0] == -1
    assert _status([_deep(0, 4, 8, 2)], 16)[0] == -1
    assert _status([_deep(4, 0, 8, 2)], 16)[0] == -1
    assert _status([_deep(9, 8, 8, 2)], 16)[0] == -1  # n1 + n2 > D
    for missing in ("p0", "p1", "p2", "i0", "i1"):
        assert _status([_deep(4, 4, 8, 2, **{missing: None})], 16)[0] == -1, missing
    assert _status([_deep(4, 4, 8, 2, c=False)], 16)[0] == 0  # c is optional


def test_float64_entry_points_refuse_the_kind():
    from bijectors_jl_b200 import _lib

    a = _arr([_deep(4, 4, 8, 3)], _lib.LayerDesc64)
    L_ = _lib.lib()
    assert L_.b2b_chain_vjp_workspace_bytes_f64(a, 1, 16, 1000) == 0
    assert L_.b2b_chain_vjp_f64(a, 1, None, None, None, None, None, 16, 0, 16, 16, 16, None, 0, None) == -2


def test_mixed_chain_plans():
    """With planar, BatchNorm, Permute and one-hidden-layer neighbours and a terminal MvNormal: accepted, no forward
    workspace, and the VJP workspace holds one checkpoint per extra segment."""
    from bijectors_jl_b200 import _lib

    D, N = 64, 1 << 20
    planar = dict(kind=_lib.PLANAR, p0=P, p1=P, p2=P)
    bn = dict(kind=_lib.BATCHNORM, p0=P, p1=P, p2=P, p3=P, f0=1e-5)
    perm = dict(kind=_lib.PERMUTE, i0=P)
    diag = dict(kind=_lib.MVNORMAL_DIAG, p0=P, p1=P)
    mlp = dict(kind=_lib.COUPLING_MLP, p0=P, p1=P, p2=P, p3=P, i0=P, i1=P, n0=32, n1=32, n2=64, n3=0)
    deep = _deep(32, 32, 64, 3)
    chain = [planar, bn, deep, bn, perm, mlp, _deep(32, 32, 64, 2, act=1, inv=1), diag]
    st, fwd, vjp = _status(chain, D)
    assert st == 0 and fwd == 0
    L_ = _lib.lib()
    a = _arr(chain, _lib.LayerDesc)
    assert L_.b2b_chain_workspace_bytes(a, len(chain), D, N, 0, 0) >= D * N * 4
    assert vjp > _status([deep], D)[2] + 4 * D * N * 4
