"""Tests of B2B_ELEMENTWISE_VEC (Shift / Scale / LeakyReLU with a trainable vector) that need no GPU: the float64 reference
against central differences, the constants of the header and both bindings, the descriptor rules through the host paths
(N = 0 calls and workspace queries), the Python layer, and the SASS of the x̄-only elementwise-run kernels."""
import ctypes
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import elementwise_vec_oracle as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAWS = (E.SHIFT, E.SCALE, E.LEAKY_RELU)


@pytest.fixture(scope="module")
def B():
    import bijectors_jl_b200 as B

    return B


def param(law, D, rng):
    if law == E.SCALE:
        return rng.uniform(0.5, 2.0, D) * rng.choice([-1.0, 1.0], D)
    return rng.uniform(0.2, 2.0, D) if law == E.LEAKY_RELU else rng.standard_normal(D)


# ---- the reference ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("law", LAWS)
def test_oracle_against_central_differences(law, inverse):
    rng = np.random.default_rng(law * 2 + inverse)
    D, N, h = 6, 9, 1e-6
    a = param(law, D, rng)
    x = rng.standard_normal((D, N))
    x = np.where(np.abs(x) < 0.05, 0.3, x)  # away from LeakyReLU's kink
    ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal(N)

    def J(av, xv):
        y, lj = E.VecLayer(law, av)._apply(xv, inverse)
        return float((ybar * y).sum() + (ljbar * lj).sum())

    lay = E.VecLayer(law, a)
    xb, g = lay.vjp(x, ybar, ljbar, inverse)
    fx = np.zeros_like(x)
    for i in range(D):
        for n in range(N):
            e = np.zeros_like(x)
            e[i, n] = h
            fx[i, n] = (J(a, x + e) - J(a, x - e)) / (2 * h)
    fa = np.array([(J(a + h * np.eye(D)[i], x) - J(a - h * np.eye(D)[i], x)) / (2 * h) for i in range(D)])
    assert np.abs(fx - xb).max() <= 1e-7 * max(1.0, np.abs(fx).max())
    assert np.abs(fa - g[lay.name]).max() <= 1e-7 * max(1.0, np.abs(fa).max())
    # the inverse undoes the forward
    y, lj = lay.forward(x)
    xi, lji = lay.inverse(y)
    assert np.allclose(xi, x, atol=1e-12) and np.allclose(lji, -lj, atol=1e-12)


@pytest.mark.parametrize("inverse", [False, True])
def test_chain_oracle_against_central_differences(inverse):
    """elementwise_vec_oracle.chain_vjp through Permute, Scale(a) and Shift(b): ā, b̄ and x̄ against central differences."""
    import chain_vjp_oracle as V
    from oracle import oracle_np as O

    rng = np.random.default_rng(7 + inverse)
    D, N, h = 6, 11, 1e-6
    perm = (rng.permutation(D) + 1).tolist()
    a, b = param(E.SCALE, D, rng), param(E.SHIFT, D, rng)
    x, ybar, ljbar = rng.standard_normal((D, N)), rng.standard_normal((D, N)), rng.standard_normal(N)
    flags = [inverse] * 3

    def layers(av, bv):
        return [O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))), E.VecLayer(E.SCALE, av),
                E.VecLayer(E.SHIFT, bv)]

    def J(av, bv, xv):
        y, lj = V.chain_logjac(layers(av, bv), flags, xv)
        return float((ybar * y).sum() + (ljbar * lj).sum())

    xb, grads, _ = E.chain_vjp(layers(a, b), flags, x, ybar, ljbar)
    I = np.eye(D)
    fa = np.array([(J(a + h * I[i], b, x) - J(a - h * I[i], b, x)) / (2 * h) for i in range(D)])
    fb = np.array([(J(a, b + h * I[i], x) - J(a, b - h * I[i], x)) / (2 * h) for i in range(D)])
    fx = np.array([[(J(a, b, x + h * np.outer(I[i], np.eye(N)[n])) - J(a, b, x - h * np.outer(I[i], np.eye(N)[n]))) / (2 * h)
                    for n in range(N)] for i in range(D)])
    for got, want in ((grads[1]["a"], fa), (grads[2]["a"], fb), (xb, fx)):
        assert np.abs(got - want).max() <= 1e-7 * max(1.0, np.abs(want).max())


# ---- constants ----------------------------------------------------------------------------------------------------------
def test_constants_agree(B):
    hdr = open(os.path.join(ROOT, "include", "b2b.h")).read()
    jl = open(os.path.join(ROOT, "bijectors.jl_b200", "julia", "B200Bijectors.jl")).read()
    assert int(re.search(r"#define B2B_ELEMENTWISE_VEC (\d+)", hdr).group(1)) == B._lib.ELEMENTWISE_VEC == 17
    assert int(re.search(r"const ELEMENTWISE_VEC = Int32\((\d+)\)", jl).group(1)) == 17
    for name, v in (("SHIFT", E.SHIFT), ("SCALE", E.SCALE), ("LEAKY_RELU", E.LEAKY_RELU)):
        assert int(re.search(rf"#define B2B_EW_{name} (\d+)", hdr).group(1)) == v == getattr(B._lib, f"EW_{name}")


# ---- descriptor rules through the host paths ----------------------------------------------------------------------------
def descs(B, law=E.SCALE, D=8, p0=0x1000, f64=False, n=1):
    d = (B._lib.LayerDesc64 if f64 else B._lib.LayerDesc)()
    d.kind, d.n0, d.p0 = B._lib.ELEMENTWISE_VEC, law, p0
    return (type(d) * n)(*([d] * n))


def vjp_status(B, arr, D, bars=None, L=1, f64=False):
    fn = B.lib().b2b_chain_vjp_f64 if f64 else B.lib().b2b_chain_vjp_f32
    pb = None
    if bars is not None:
        ptrs = (ctypes.c_void_p * (4 * L))(*bars)
        pb = ctypes.cast(ptrs, ctypes.c_void_p)
    return fn(arr, L, 0x2000, None, None, 0x3000, pb, D, 0, D, D, D, None, 0, None)


def test_status_codes(B):
    lib, L_ = B.lib(), B._lib
    assert vjp_status(B, descs(B), 8) == L_.B2B_OK
    assert lib.b2b_chain_vjp_workspace_bytes(descs(B), 1, 8, 1000) > 0
    assert vjp_status(B, descs(B, p0=None), 8) == L_.B2B_EINVAL
    for bad in (0, 1, 2, 6, 7, 8, -1):
        assert vjp_status(B, descs(B, law=bad), 8) == L_.B2B_EINVAL, bad
        assert lib.b2b_chain_vjp_workspace_bytes(descs(B, law=bad), 1, 8, 1000) == 0
    for slot in (1, 2, 3):
        bars = [None] * 4
        bars[slot] = 0x4000
        assert vjp_status(B, descs(B), 8, bars) == L_.B2B_EUNSUPPORTED, slot
    assert vjp_status(B, descs(B, D=1025), 1025) == L_.B2B_EUNSUPPORTED
    assert lib.b2b_chain_vjp_workspace_bytes(descs(B), 1, 1025, 1000) == 0
    assert lib.b2b_chain_vjp_workspace_bytes(descs(B), 1, 1024, 1000) > 0
    # the Float64 entry points take the kind
    assert lib.b2b_chain_vjp_workspace_bytes_f64(descs(B, f64=True), 1, 8, 1000) > 0
    assert vjp_status(B, descs(B, f64=True), 8, f64=True) == L_.B2B_OK
    assert vjp_status(B, descs(B, law=1, f64=True), 8, f64=True) == L_.B2B_EINVAL


def test_workspace_grows_only_with_the_kind(B):
    """A run with V vector layers adds G·V·D floats to the workspace of the same run of STACKED_EW layers."""
    lib, L_ = B.lib(), B._lib
    D, N = 64, 4096

    def run(kinds):
        arr = (L_.LayerDesc * len(kinds))()
        for d, k in zip(arr, kinds):
            d.kind = k
            d.n0, d.p0, d.i0 = E.SCALE, 0x1000, 0x2000
        return lib.b2b_chain_vjp_workspace_bytes(arr, len(kinds), D, N)

    S, V, M = L_.STACKED_EW, L_.ELEMENTWISE_VEC, L_.MVNORMAL_DIAG
    base, one, two = run([S, S, M]), run([S, V, M]), run([V, V, M])
    assert run([S, S]) == 256 and run([S, V]) > 256  # 256: the alignment slack of every chain workspace
    step = one - base
    assert step > 0 and two - one == step and step % (4 * D) == 0
    assert run([S, V]) == step + 512  # the kernel slice and the chain workspace each keep 256 bytes of alignment slack


# ---- the Python layer ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls,law,name", [("Shift", E.SHIFT, "a"), ("Scale", E.SCALE, "a"), ("LeakyReLU", E.LEAKY_RELU, "α")])
def test_python_layer(B, cls, law, name):
    from bijectors_jl_b200.autograd import _trainable_tensors
    from bijectors_jl_b200.interface import _slot_names

    C = getattr(B, cls)
    a = np.linspace(0.5, 1.5, 5)
    lay = C(a, device="cpu")
    assert lay.vector and lay.a.dtype == torch.float32 and lay.a.shape == (5,)
    (d,) = lay._descs(False, 5)
    assert (d.kind, d.n0, d.inverse, d.p0, d.p1, d.i0) == (B._lib.ELEMENTWISE_VEC, law, 0, lay.a.data_ptr(), None, None)
    assert _slot_names(d) == (name,)
    inv = B.inverse(lay)
    assert isinstance(inv, B.Inverse) and inv.orig is lay and inv._descs(False, 5)[0].inverse == 1
    with pytest.raises(ValueError, match="DimensionMismatch"):
        lay._descs(False, 6)
    with pytest.raises(B.B2BError) as e:
        B.Stacked([lay], [(1, 5)], device="cpu")
    assert e.value.status == B._lib.B2B_EUNSUPPORTED
    assert _trainable_tensors(lay) == [lay.a] and _trainable_tensors(inv) == [lay.a]
    assert lay._keepalive() == (lay.a,)
    assert lay == C(torch.tensor(a), device="cpu") and lay != C(a * 2, device="cpu") and lay != C(1.0)
    d64 = C(a, device="cpu", dtype=torch.float64)._descs(False, 5, torch.float64)[0]
    assert isinstance(d64, B._lib.LayerDesc64) and d64.kind == B._lib.ELEMENTWISE_VEC
    with pytest.raises(TypeError):
        C(a, device="cpu", dtype=torch.float64)._descs(False, 5, torch.float32)
    # scalars and 0-d values stay the STACKED_EW row law, with no trainable tensor
    for s in (0.7, np.float32(0.7), np.array(0.7), torch.tensor(0.7)):
        sc = C(s)
        assert not sc.vector and sc.a == pytest.approx(0.7) and _trainable_tensors(sc) == [] and sc._keepalive() == ()


def test_scalar_inverses_unchanged(B):
    assert B.inverse(B.Shift(0.5)) == B.Shift(-0.5)
    assert B.inverse(B.LeakyReLU(0.5)) == B.LeakyReLU(2.0)
    assert isinstance(B.inverse(B.Scale(0.5)), B.Inverse)


def test_leaky_relu_needs_positive_slopes(B):
    with pytest.raises(ValueError):
        B.LeakyReLU(np.array([0.5, 0.0, 1.0]), device="cpu")
    with pytest.raises(ValueError):
        B.LeakyReLU(-0.1)


# ---- SASS of the x̄-only instantiations ----------------------------------------------------------------------------------
def test_existing_ew_vjp_kernels_keep_their_sass():
    """ew_vjp_kernel<256, 4> and <1024, 2> compile to the instructions they had before ELEMENTWISE_VEC (fingerprints taken
    with the nvcc recorded next to them; another compiler version is not comparable)."""
    obj = os.path.join(ROOT, "bijectors.jl_b200", "csrc", "b2b_ew_vjp.o")
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "ew_vjp_sass.json")))
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not (os.path.exists(obj) and os.path.exists(cuobjdump) and os.path.exists(nvcc)):
        pytest.skip("needs the built object and the CUDA toolkit")
    if subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1] != gold["nvcc"]:
        pytest.skip("another nvcc version")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur and re.search(r"/\*[0-9a-f]{4}\*/", line):
            funcs[cur].append(re.sub(r"\s+", " ", line.strip()))
    for name, digest in gold["sha256"].items():
        assert hashlib.sha256("\n".join(funcs[name]).encode()).hexdigest() == digest, name
