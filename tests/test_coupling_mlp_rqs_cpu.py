"""CPU tests of the neural spline coupling reference (tests/coupling_mlp_rqs_oracle.py) and of the host-side pieces of
B2B_COUPLING_MLP_RQS: the oracle's reverse mode against central differences, its log-Jacobian against log|det J| of a
finite-difference Jacobian, the inverse, the collapse to the linear spline coupling at LeakyReLU slope 1 and at W₂ = 0,
the constructor's errors, the descriptor fields, the constants of the three bindings, and -- with fake pointers at N = 0,
as test_coupling_mlp_cpu.py does it -- the status codes and workspace sizes of the chain entry points around the
envelope."""
import os
import re

import numpy as np
import pytest

import coupling_mlp_rqs_oracle as R
import spline_coupling_oracle as S

ROOT = os.path.join(os.path.dirname(__file__), "..")
P = 0x10000  # a fake device address: nothing is read through it
ACTS = [("tanh", 0.0), ("leaky_relu", 0.2)]


def _case(rng, n1, n2, H, K, scale=0.7):
    J = 3 * K - 1
    return (rng.standard_normal((H, n2)) * scale, rng.standard_normal(H) * 0.5,
            rng.standard_normal((J * n1, H)) * scale / np.sqrt(H), rng.standard_normal(J * n1) * 0.3)


def _fd(f, a, h=1e-6):
    g = np.zeros_like(a)
    for i in np.ndindex(a.shape):
        p, m = a.copy(), a.copy()
        p[i] += h
        m[i] -= h
        g[i] = (f(p) - f(m)) / (2 * h)
    return g


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
def test_vjp_matches_central_differences(inv, act, slope):
    rng = np.random.default_rng(3 + inv + len(act))
    D, N, H, K, B = 6, 4, 4, 3, 2.0
    idx1, idx2 = [2, 5], [6, 3, 1]  # row 4 is an x₃ row
    W1, c1, W2, c2 = _case(rng, len(idx1), len(idx2), H, K)
    x = rng.standard_normal((D, N)) * 0.8
    x[1, 0] = 3.0  # one element outside the box: the identity
    yb, lb = rng.standard_normal((D, N)), rng.standard_normal(N)
    f = R.inverse if inv else R.forward

    def loss(x_, W1_, c1_, W2_, c2_):
        y, lj = f(idx1, idx2, W1_, c1_, W2_, c2_, K, B, act, slope, x_)
        return float(np.sum(y * yb) + np.sum(lj * lb))

    xb, g = R.vjp(idx1, idx2, W1, c1, W2, c2, K, B, act, slope, x, yb, lb, inverse=inv)
    args = [x, W1, c1, W2, c2]
    for k, got in enumerate((xb, g["W1"], g["c1"], g["W2"], g["c2"])):
        want = _fd(lambda a: loss(*(args[:k] + [a] + args[k + 1:])), args[k])
        assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max()), k


@pytest.mark.parametrize("act,slope", ACTS)
def test_logjac_is_log_det_of_the_jacobian_and_inverse_undoes_forward(act, slope):
    rng = np.random.default_rng(4)
    D, H, K, B = 5, 3, 4, 3.0
    idx1, idx2 = [1, 4], [2, 5]
    W1, c1, W2, c2 = _case(rng, 2, 2, H, K)
    x = rng.standard_normal(D)
    for f in (R.forward, R.inverse):
        def col(v):
            return f(idx1, idx2, W1, c1, W2, c2, K, B, act, slope, v[:, None])[0][:, 0]

        Jm = np.stack([(col(x + h) - col(x - h)) / 2e-6 for h in np.eye(D) * 1e-6], axis=1)
        lj = f(idx1, idx2, W1, c1, W2, c2, K, B, act, slope, x[:, None])[1][0]
        assert abs(np.log(abs(np.linalg.det(Jm))) - lj) < 1e-6
    X = rng.standard_normal((D, 40)) * 1.5
    y, lj = R.forward(idx1, idx2, W1, None, W2, c2, K, B, act, slope, X)
    xr, ljr = R.inverse(idx1, idx2, W1, None, W2, c2, K, B, act, slope, y)
    np.testing.assert_allclose(xr, X, atol=1e-10, rtol=0)
    np.testing.assert_allclose(ljr, -lj, atol=1e-10, rtol=0)
    assert np.array_equal(y[[1, 2, 4]], X[[1, 2, 4]])


def test_slope_one_is_the_linear_spline_coupling_and_tanh_is_not():
    """LeakyReLU(1) is the identity, so the layer is COUPLING_RQS on W = W₂W₁, c = W₂c₁ + c₂."""
    rng = np.random.default_rng(8)
    D, N, H, K, B = 6, 9, 4, 5, 2.5
    idx1, idx2 = [1, 3], [2, 6, 5]
    W1, c1, W2, c2 = _case(rng, 2, 3, H, K)
    x = rng.standard_normal((D, N))
    ya, la = S.forward(idx1, idx2, W2 @ W1, W2 @ c1 + c2, K, B, x)
    y, lj = R.forward(idx1, idx2, W1, c1, W2, c2, K, B, "leaky_relu", 1.0, x)
    np.testing.assert_allclose(y, ya, atol=1e-12, rtol=0)
    np.testing.assert_allclose(lj, la, atol=1e-12, rtol=0)
    yt, lt = R.forward(idx1, idx2, W1, c1, W2, c2, K, B, "tanh", 0.0, x)
    assert np.abs(yt - ya).max() > 1e-3 and np.abs(lt - la).max() > 1e-3


def test_zero_last_layer_is_the_spline_of_c2():
    rng = np.random.default_rng(9)
    D, N, H, K, B = 5, 7, 3, 4, 3.0
    idx1, idx2 = [2, 3], [1, 5]
    W1, c1, W2, c2 = _case(rng, 2, 2, H, K)
    x = rng.standard_normal((D, N))
    y, lj = R.forward(idx1, idx2, W1, c1, np.zeros_like(W2), c2, K, B, "tanh", 0.0, x)
    ya, la = S.forward(idx1, idx2, np.zeros((W2.shape[0], 2)), c2, K, B, x)
    np.testing.assert_allclose(y, ya, atol=1e-12, rtol=0)
    np.testing.assert_allclose(lj, la, atol=1e-12, rtol=0)


def test_conditioner_errors_and_descriptor():
    import torch

    import bijectors_jl_b200 as B
    from bijectors_jl_b200 import _lib

    H, n1, n2, K = 5, 3, 2, 4
    J = 3 * K - 1
    z = lambda *s: np.zeros(s, np.float32)  # noqa: E731
    ok = dict(K=K, B=2.0, device="cpu")
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(H, n2), None, z(J * n1 + 1, H), None, **ok)  # rows not a multiple of 3K − 1
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(H, n2), None, z(J * n1, H + 1), None, **ok)  # W2's columns are not H
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(H, n2), z(H + 1), z(J * n1, H), None, **ok)
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(H, n2), None, z(J * n1, H), z(J * n1 - 1), **ok)
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(H, n2), None, z(J * n1, H), None, activation="gelu", **ok)
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(H, n2), None, z(J * n1, H), None, K=0, B=2.0, device="cpu")
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(H, n2), None, z(J * n1, H), None, K=K, B=0.0, device="cpu")
    with pytest.raises(ValueError):
        B.MLPSplineConditioner(z(0, n2), None, z(J * n1, 0), None, **ok)
    with pytest.raises(TypeError):
        B.MLPSplineConditioner(z(H, n2), None, z(J * n1, H), None, dtype=torch.float64, **ok)
    W1 = np.arange(H * n2, dtype=np.float32).reshape(H, n2)
    W2 = np.arange(J * n1 * H, dtype=np.float32).reshape(J * n1, H)
    cond = B.MLPSplineConditioner(W1, np.ones(H, np.float32), W2, np.ones(J * n1, np.float32), K=K, B=2.5,
                                  activation="leaky_relu", slope=0.25, device="cpu")
    assert (cond.n1, cond.n2, cond.H, cond.K, cond.B) == (n1, n2, H, K, 2.5)
    assert np.array_equal(cond.W1.numpy().T, W1) and np.array_equal(cond.W2.numpy().T, W2)  # column-major storage
    mask = B.PartitionMask(7, [2, 4, 6], [1, 7])
    with pytest.raises(ValueError):
        B.Coupling(cond, B.PartitionMask(7, [2, 4], [1, 7]))
    cl = B.Coupling(cond, mask)
    d = cl._descs(True, 7)[0]
    assert (d.kind, d.inverse, d.n0, d.n1, d.n2) == (_lib.COUPLING_MLP_RQS, 1, n1, n2, H)
    assert d.n3 == _lib.ACT_LEAKY_RELU | (K << 8) and d.f0 == 0.25 and d.f1 == 2.5
    assert (d.p0, d.p1, d.p2, d.p3) == tuple(t.data_ptr() for t in (cond.W1, cond.c1, cond.W2, cond.c2))
    assert d.i0 == cl._idx1.data_ptr() and d.i1 == cl._idx2.data_ptr()
    with pytest.raises(TypeError):
        cl._descs(False, 7, torch.float64)
    bare = B.MLPSplineConditioner(W1, None, W2, None, K=K, B=2.5, device="cpu")
    nd = B.Coupling(bare, mask)._descs(False, 7)[0]
    assert nd.p1 is None and nd.p3 is None and nd.n3 == _lib.ACT_TANH | (K << 8)
    assert B.coupling(cl) is cond and cl == B.Coupling(cond.to("cpu"), mask) and cl != B.Coupling(bare, mask)
    other_B = B.MLPSplineConditioner(W1, np.ones(H, np.float32), W2, np.ones(J * n1, np.float32), K=K, B=3.0,
                                     activation="leaky_relu", slope=0.25, device="cpu")
    assert cl != B.Coupling(other_B, mask)
    assert [t.data_ptr() for t in B.autograd._trainable_tensors(B.Coupling(bare, mask))] == [bare.W1.data_ptr(), bare.W2.data_ptr()]
    assert len(B.autograd._trainable_tensors(cl)) == 4
    with pytest.raises(B.B2BError, match="MLPSplineConditioner"):
        B.Coupling(object(), mask)


def test_header_python_and_julia_constants_agree():
    from bijectors_jl_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    jl = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()

    def define(name):
        return int(re.search(rf"#define B2B_{name} (\d+)", hdr).group(1))

    assert define("COUPLING_MLP_RQS") == _lib.COUPLING_MLP_RQS == 14 and "const COUPLING_MLP_RQS = Int32(14)" in jl
    assert tuple(define(f"COUPLING_MLP_RQS_MAX_{s}") for s in "NHKD") == \
        (_lib.COUPLING_MLP_RQS_MAX_N, _lib.COUPLING_MLP_RQS_MAX_H, _lib.COUPLING_MLP_RQS_MAX_K,
         _lib.COUPLING_MLP_RQS_MAX_D) == (128, 128, 16, 1024)
    kinds = {int(v) for v in re.findall(r"#define B2B_[A-Z_]+ (\d+) +/\* [A-Z]", hdr)}
    assert 14 in kinds and 10 not in kinds


# ---- the chain entry points on the host --------------------------------------------------------------------------------
def _nsf(n1, n2, H, K, act=0, inv=0, c=True, **over):
    from bijectors_jl_b200 import _lib

    d = dict(kind=_lib.COUPLING_MLP_RQS, inverse=inv, p0=P, p2=P, i0=P, i1=P, n0=n1, n1=n2, n2=H, n3=act | (K << 8),
             f0=0.1, f1=3.0)
    if c:
        d.update(p1=P, p3=P)
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


@pytest.mark.parametrize("n1,n2,H,K,D", [(1, 1, 1, 2, 3), (3, 4, 7, 5, 10), (128, 128, 128, 16, 256),
                                         (128, 128, 128, 16, 1024)])
def test_inside_the_envelope(n1, n2, H, K, D):
    for act in (0, 1):
        for inv in (0, 1):
            for c in (True, False):
                st, fwd, vjp = _status([_nsf(n1, n2, H, K, act, inv, c)], D)
                assert st == 0 and fwd == 0 and vjp > 0  # the forward launch needs no workspace
                # two D x N cotangent buffers, plus the slices of the parameter sums: those stay under 256 MiB
                assert 0 < vjp - 2 * D * (1 << 20) * 4 <= (256 << 20) + (1 << 20)


@pytest.mark.parametrize("n1,n2,H,K,D", [(129, 1, 4, 4, 300), (1, 129, 4, 4, 300), (4, 4, 129, 4, 40),
                                         (4, 4, 4, 17, 40), (4, 4, 4, 4, 1025), (4, 4, 4, 1, 40)])
def test_just_past_the_envelope(n1, n2, H, K, D):
    assert _status([_nsf(n1, n2, H, K)], D) == (-2, 0, 0)


def test_invalid_descriptors():
    assert _status([_nsf(4, 4, 8, 4, act=2)], 16)[0] == -1
    assert _status([_nsf(4, 4, 8, 4, act=255)], 16)[0] == -1
    assert _status([_nsf(4, 4, 8, 0)], 16)[0] == -1
    assert _status([_nsf(4, 4, 8, 4, f1=0.0)], 16)[0] == -1
    assert _status([_nsf(4, 4, 8, 4, f1=-1.0)], 16)[0] == -1
    assert _status([_nsf(4, 4, 0, 4)], 16)[0] == -1
    assert _status([_nsf(0, 4, 8, 4)], 16)[0] == -1
    assert _status([_nsf(4, 0, 8, 4)], 16)[0] == -1
    assert _status([_nsf(9, 8, 8, 4)], 16)[0] == -1  # n1 + n2 > D
    for missing in ("p0", "p2", "i0", "i1"):
        assert _status([_nsf(4, 4, 8, 4, **{missing: None})], 16)[0] == -1, missing


def test_float64_entry_points_refuse_the_kind():
    from bijectors_jl_b200 import _lib

    a = _arr([_nsf(4, 4, 8, 4)], _lib.LayerDesc64)
    L_ = _lib.lib()
    assert L_.b2b_chain_vjp_workspace_bytes_f64(a, 1, 16, 1000) == 0
    assert L_.b2b_chain_vjp_f64(a, 1, None, None, None, None, None, 16, 0, 16, 16, 16, None, 0, None) == -2


def test_mixed_chain_plans():
    """With planar, BatchNorm and Permute neighbours and a terminal MvNormal: accepted, no forward workspace, and the
    VJP workspace holds one checkpoint per extra segment."""
    from bijectors_jl_b200 import _lib

    D, N = 64, 1 << 20
    planar = dict(kind=_lib.PLANAR, p0=P, p1=P, p2=P)
    bn = dict(kind=_lib.BATCHNORM, p0=P, p1=P, p2=P, p3=P, f0=1e-5)
    perm = dict(kind=_lib.PERMUTE, i0=P)
    diag = dict(kind=_lib.MVNORMAL_DIAG, p0=P, p1=P)
    nsf = _nsf(32, 32, 64, 8)
    chain = [planar, bn, nsf, bn, perm, _nsf(32, 32, 64, 8, act=1, inv=1), diag]
    st, fwd, vjp = _status(chain, D)
    assert st == 0 and fwd == 0
    L_ = _lib.lib()
    a = _arr(chain, _lib.LayerDesc)
    assert L_.b2b_chain_workspace_bytes(a, len(chain), D, N, 0, 0) >= D * N * 4
    assert vjp > _status([nsf], D)[2] + 4 * D * N * 4
