"""Reparameterised sampling without a device: the C prototypes, the float64 cotangent formulas of tests/rsample_oracle.py
against central differences of (y, log q), and the argument checks that run before anything is launched."""
import ctypes
import os
import re

import numpy as np
import pytest

import mvnormal_tril_oracle as T
import rsample_oracle as R
from oracle import oracle_np as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["b2b_chain_sample_logq_workspace_bytes", "b2b_chain_sample_logq_f32", "b2b_chain_sample_vjp_workspace_bytes",
       "b2b_chain_sample_vjp_f32"]


def header_args(name):
    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", NEW)
def test_prototypes_match_header(name):
    import bijectors_jl_b200._lib as lib

    res, args = lib._SIGS[name]
    hargs = header_args(name)
    assert len(args) == len(hargs), (name, len(args), len(hargs))
    for a, h in zip(args, hargs):
        if "b2b_layer_desc*" in h.replace(" *", "*"):
            assert a is not ctypes.c_void_p and "LayerDesc" in repr(a), (name, h)
        elif "*" in h:
            assert a is ctypes.c_void_p, (name, h)
        elif h.startswith("int32_t"):
            assert a is ctypes.c_int32, (name, h)
        elif h.startswith("int64_t"):
            assert a is ctypes.c_int64, (name, h)
        elif h.startswith("uint64_t"):
            assert a is ctypes.c_uint64, (name, h)
        elif h.startswith("size_t"):
            assert a is ctypes.c_size_t, (name, h)
    assert res is (ctypes.c_size_t if name.endswith("_bytes") else ctypes.c_int)


def test_julia_wrappers_call_the_new_entry_points():
    src = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()
    for name in NEW:
        assert f":{name}" in src, name


# ---- the cotangent formulas against central differences -----------------------------------------------------------
def layers(rng, D):
    f = np.float64
    pl = [O.Layer("planar", dict(w=rng.standard_normal(D) * 0.4, u=rng.standard_normal(D) * 0.4, b=rng.standard_normal(1)))
          for _ in range(2)]
    K = 5
    spl = O.Layer("rqs", dict(widths=np.sort(rng.uniform(-3, 3, (D, K + 1)), axis=1).astype(f),
                              heights=np.sort(rng.uniform(-3, 3, (D, K + 1)), axis=1).astype(f),
                              derivs=rng.uniform(0.5, 2.0, (D, K + 1)).astype(f)))
    spl.params["derivs"][:, 0] = spl.params["derivs"][:, -1] = 1.0
    st = O.Layer("stacked", dict(ops=[(O.EW.SHIFT, 0.4), (O.EW.SCALE, -1.2)], ranges=[(1, 2), (3, D)]))
    return [pl[0], spl, st, pl[1]], [False, False, False, True]


def objective(ol, flags, z, ybar, qbar, mu, sigma, L):
    y, lq = R.forward(ol, flags, z, mu, sigma, L)
    return float(np.sum(ybar * y) + np.sum(qbar * lq))


@pytest.mark.parametrize("base", ["diag", "tril"])
@pytest.mark.parametrize("chain", ["none", "mixed"])
def test_cotangents_match_central_differences(base, chain):
    rng = np.random.default_rng(7 + len(base) + len(chain))
    D, N, h = 5, 6, 1e-6
    ol, flags = layers(rng, D) if chain == "mixed" else ([], [])
    z = rng.standard_normal((D, N))
    ybar, qbar = rng.standard_normal((D, N)), rng.standard_normal(N)
    mu = rng.standard_normal(D) * 0.3
    sigma = rng.uniform(0.6, 1.4, D) if base == "diag" else None
    L = T.random_tril(rng, D) if base == "tril" else None
    grads, bg = R.vjp(ol, flags, z, ybar, qbar, mu, sigma, L)

    def fd(arr, idx, f):
        old = arr[idx]
        arr[idx] = old + h
        a = f()
        arr[idx] = old - h
        b = f()
        arr[idx] = old
        return (a - b) / (2 * h)

    J = lambda: objective(ol, flags, z, ybar, qbar, mu, sigma, L)
    for i in range(D):
        assert abs(fd(mu, i, J) - bg["μ"][i]) <= 1e-6 * max(1.0, abs(bg["μ"][i]))
        if sigma is not None:
            assert abs(fd(sigma, i, J) - bg["σ"][i]) <= 1e-6 * max(1.0, abs(bg["σ"][i]))
    if L is not None:
        for i in range(D):
            for j in range(D):
                g = fd(L, (i, j), J) if i >= j else 0.0
                assert abs(g - bg["L"][i, j]) <= 1e-6 * max(1.0, abs(bg["L"][i, j])), (i, j)
    if chain == "mixed":
        for l, name, key in [(0, "w", "w"), (0, "u", "u"), (3, "w", "w"), (1, "widths", "widths")]:
            arr = ol[l].params[name]
            for idx in [(0,), (D - 1,)] if arr.ndim == 1 else [(0, 2), (D - 1, 3)]:
                got = np.reshape(grads[l][key], arr.shape)[idx]
                assert abs(fd(arr, idx, J) - got) <= 1e-5 * max(1.0, abs(got)), (l, name, idx)


# ---- argument checks before any launch -------------------------------------------------------------------------------
def test_float64_flow_or_base_raises():
    import torch

    import bijectors_jl_b200 as B

    base64 = B.MvNormal(4, mu=np.zeros(4), sigma=np.ones(4), device="cpu", dtype=torch.float64)
    with pytest.raises(TypeError):
        B.rand_logpdf(base64, 3, seed=1)
    with pytest.raises(TypeError):
        B.rand_vjp(base64, 3, seed=1)
    tril64 = B.MvNormal(4, scale_tril=np.eye(4), device="cpu", dtype=torch.float64)
    with pytest.raises(TypeError):
        B.rand_logpdf(tril64, 3, seed=1)


def test_bad_base_kind_and_chain_are_refused():
    import bijectors_jl_b200 as B
    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200._lib import LayerDesc

    lib = B.lib()
    base = (LayerDesc * 1)()
    for kind in (_lib.PLANAR, 10, _lib.MVNORMAL_DIAG + 100):
        base[0].kind = kind
        assert lib.b2b_chain_sample_logq_workspace_bytes(None, 0, base, 8, 100) == 0
        assert lib.b2b_chain_sample_vjp_workspace_bytes(None, 0, base, 8, 100) == 0
        assert lib.b2b_chain_sample_logq_f32(None, 0, base, 1, 0, 0, None, None, 8, 100, 8, None, 0, None) == _lib.B2B_EINVAL
        assert lib.b2b_chain_sample_vjp_f32(None, 0, base, 1, 0, 0, None, 8, None, None, 8, 100, None, 0, None) == \
            _lib.B2B_EINVAL
        assert lib.b2b_last_launch_count() == 0
    base[0].kind = _lib.MVNORMAL_DIAG
    assert lib.b2b_chain_sample_logq_workspace_bytes(None, 0, base, 8, 100) > 0
    assert lib.b2b_chain_sample_vjp_workspace_bytes(None, 0, base, 8, 100) > 0
    base[0].kind = _lib.MVNORMAL_TRIL  # L is required
    assert lib.b2b_chain_sample_vjp_workspace_bytes(None, 0, base, 8, 100) == 0
    base[0].p1 = 16
    assert lib.b2b_chain_sample_vjp_workspace_bytes(None, 0, base, 8, 100) > 0
    assert lib.b2b_chain_sample_vjp_workspace_bytes(None, 0, base, 257, 100) == 0
    assert lib.b2b_chain_sample_logq_f32(None, 0, base, 1, 0, 0, None, None, 257, 100, 257, None, 0, None) == \
        _lib.B2B_EUNSUPPORTED
    # a chain holding a terminal, and a planar layer past its reverse-mode kernels (D > 128)
    term = (LayerDesc * 1)()
    term[0].kind = _lib.MVNORMAL_DIAG
    assert lib.b2b_chain_sample_vjp_workspace_bytes(term, 1, base, 8, 100) == 0
    pl = (LayerDesc * 1)()
    pl[0].kind, pl[0].p0, pl[0].p1, pl[0].p2 = _lib.PLANAR, 16, 32, 48
    assert lib.b2b_chain_sample_vjp_workspace_bytes(pl, 1, base, 64, 100) > 0
    base[0].kind, base[0].p1 = _lib.MVNORMAL_DIAG, None
    assert lib.b2b_chain_sample_vjp_workspace_bytes(pl, 1, base, 300, 100) == 0
    assert lib.b2b_chain_sample_logq_f32(pl, 1, base, 1, 0, 0, None, None, 300, 100, 300, None, 0, None) == \
        _lib.B2B_EUNSUPPORTED
