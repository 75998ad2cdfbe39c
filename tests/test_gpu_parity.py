"""GPU parity tests proper: the CUDA path (through the C ABI) against the oracle on identical seeded inputs.

Tolerance (north_star): Float32 layers within 1e-5 RELATIVE of the reference CPU path, measured norm-wise
(`‖a−b‖ ≤ rtol·max(‖a‖,‖b‖)` -- the semantics of Julia's `≈` on arrays that the reference's own tests use);
index movement (Permute / PartitionMask / Stacked ranges) bit-exact.
"""
import math

import numpy as np
import pytest

from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

import os as _os

ROOT_DIR = _os.path.dirname(_os.path.dirname(_os.path.abspath(__file__)))

RTOL = 1e-5


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(o32, o64, k=2.0):
    """The parity gate of north_star: 1e-5 relative -- or, where the float32 restatement of the REFERENCE itself is
    further than that from float64 on the very same input (an ill-conditioned case), k <= 2 times the reference's own
    error.  Never a blanket multiple of the tolerance."""
    return max(RTOL, k * rel(o32, o64))


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


f32 = np.float32


def make_case(kind, D, rng):
    """(device layer, oracle layer) with float32 parameters."""
    import bijectors_jl_b200 as B

    if kind == "planar":
        w, u, b = (rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32), rng.standard_normal(1).astype(f32)
        return B.PlanarLayer(w, u, b), O.Layer("planar", dict(w=w, u=u, b=b))
    if kind == "planar_randn":  # reference default init randn(dims): saturates tanh at large D (stress variant)
        w, u, b = rng.standard_normal(D).astype(f32), rng.standard_normal(D).astype(f32), rng.standard_normal(1).astype(f32)
        return B.PlanarLayer(w, u, b), O.Layer("planar", dict(w=w, u=u, b=b))
    if kind == "radial":
        a, be, z0 = rng.standard_normal(1).astype(f32), rng.standard_normal(1).astype(f32), rng.standard_normal(D).astype(f32)
        return B.RadialLayer(a, be, z0), O.Layer("radial", dict(alpha_raw=a, beta=be, z0=z0))
    if kind == "rqs":
        K, Bx = 8, 3.0
        rw, rh, rd = rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K - 1)).astype(f32)
        lay = B.RationalQuadraticSpline(rw, rh, rd, Bx)
        W, H, Dv = lay.knots()
        return lay, O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv))
    if kind == "batchnorm":
        b, logs, m = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
        v = rng.uniform(0.5, 1.5, D).astype(f32)
        return (B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v),
                O.Layer("batchnorm", dict(bn=O.BatchNormParams(b, logs, m, v, f32(1e-5), f32(0.1)))))
    if kind == "permute":
        perm = (rng.permutation(D) + 1).tolist()
        return B.Permute(perm), O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm)))
    if kind == "coupling":
        n1 = D // 2
        mask_first = rng.integers(0, 2) == 0
        idx1 = list(range(1, n1 + 1)) if mask_first else list(range(D - n1 + 1, D + 1))
        idx2 = [i for i in range(1, D + 1) if i not in set(idx1)]
        W = (rng.standard_normal((2 * n1, len(idx2))) * 0.2 / np.sqrt(len(idx2))).astype(f32)
        c = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
        return (B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2)),
                O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c)))
    if kind == "stacked":
        r1, r2 = max(1, D // 4), max(2, D // 2)
        ranges = [(1, r1), (r1 + 1, r2), (r2 + 1, D)]
        return (B.Stacked([B.elementwise("exp"), B.Scale(-1.7), B.Shift(0.3)], ranges),
                O.Layer("stacked", dict(ops=[(O.EW.EXP, 0.0), (O.EW.SCALE, f32(-1.7)), (O.EW.SHIFT, f32(0.3))], ranges=ranges)))
    if kind == "bounded":  # Logit / TruncatedBijector blocks inside Stacked: the "bounded flow" of docs/src/flows.md:25-36
        q = max(1, D // 5)
        ranges = [(1, q), (q + 1, 2 * q), (2 * q + 1, 3 * q), (3 * q + 1, 4 * q), (4 * q + 1, D)] if D >= 5 else [(1, 1), (2, D)]
        inf = float("inf")
        bs = [B.Logit(-1.0, 3.0), B.TruncatedBijector(-1.0, inf), B.TruncatedBijector(-inf, 3.0), B.TruncatedBijector(-1.0, 3.0),
              B.TruncatedBijector(-inf, inf)][: len(ranges)]
        ops = [(O.EW.LOGIT, -1.0, 3.0), (O.EW.TRUNCATED, -1.0, inf), (O.EW.TRUNCATED, -inf, 3.0), (O.EW.TRUNCATED, -1.0, 3.0),
               (O.EW.TRUNCATED, -inf, inf)][: len(ranges)]
        return B.Stacked(bs, ranges), O.Layer("stacked", dict(ops=ops, ranges=ranges))
    if kind == "leaky_relu":  # test/bijectors/leaky_relu.jl: α = 0.1
        return B.LeakyReLU(0.1), O.Layer("stacked", dict(ops=[(O.EW.LEAKY_RELU, f32(0.1))], ranges=[(1, D)]))
    raise ValueError(kind)


KINDS = ["planar", "planar_randn", "radial", "rqs", "batchnorm", "permute", "coupling", "stacked", "leaky_relu", "bounded"]


@pytest.mark.parametrize("D,N", [(128, 1000), (64, 517), (32, 2049), (256, 300), (10, 100), (3, 7), (36, 65), (200, 33)])
@pytest.mark.parametrize("kind", KINDS)
def test_layer_forward_inverse_parity(B, kind, D, N):
    if kind in ("coupling", "stacked") and D < 3:
        pytest.skip("needs D >= 3")
    import zlib

    rng = np.random.default_rng(zlib.crc32(f"{kind}-{D}-{N}".encode()))
    lay, olay = make_case(kind, D, rng)
    scale = 1.5 if kind == "rqs" else 1.0  # ~5% of RQS inputs outside the box (identity branch)
    x = (rng.standard_normal((D, N)) * scale).astype(f32)
    if kind == "bounded":
        x = rng.uniform(-0.9, 2.9, (D, N)).astype(f32)  # inside every block's support
    xd = B.from_numpy(x)
    y, lj = B.with_logabsdet_jacobian(lay, xd)
    yo, ljo = olay.forward(x)  # float32 oracle
    yo64, ljo64 = olay.forward(x.astype(np.float64)) if kind not in ("permute",) else (yo, ljo)
    yh, ljh = B.to_numpy(y), B.to_numpy(lj)
    if kind == "permute":
        assert np.array_equal(yh.view(np.uint32), yo.view(np.uint32))  # bit-exact
        assert np.all(ljh == 0)
    else:
        assert rel(yh, yo) <= RTOL, ("y vs f32 oracle", rel(yh, yo))
        assert rel(yh, yo64) <= RTOL, ("y vs f64 oracle", rel(yh, yo64))
        # logjac: norm-wise with an absolute floor for vectors that are ~0 (e.g. saturated tanh).  The gate is
        # 1e-5, or twice the float32 reference restatement's OWN distance to float64 where that is larger
        # (only the ill-conditioned planar_randn stress variant gets there).
        lgate = gate(ljo, ljo64)
        assert np.linalg.norm(ljh - ljo64) <= lgate * max(np.linalg.norm(ljo64), math.sqrt(N) * 1e-2), (rel(ljh, ljo64), lgate)
    # transform / logabsdetjac alone agree with the fused call
    assert np.array_equal(B.to_numpy(B.transform(lay, xd)), yh)
    assert np.array_equal(B.to_numpy(B.logabsdetjac(lay, xd)), ljh)
    # inverse: ires == (x, -logjac)  (test/bijectors/utils.jl:53-62)
    xi, lji = B.with_logabsdet_jacobian(B.inverse(lay), y)
    xih, ljih = B.to_numpy(xi), B.to_numpy(lji)
    xo, ljio = olay.inverse(yh.astype(np.float64) if kind != "permute" else yh)
    if kind == "permute":
        assert np.array_equal(xih.view(np.uint32), x.view(np.uint32))
    else:
        # the float32 restatement of the reference on the SAME y: its own distance to float64 is the only thing that
        # may widen the 1e-5 gate (planar_randn: flat regions of a saturated layer are ill-conditioned to invert)
        xo32, ljio32 = olay.inverse(yh)
        assert rel(xih, xo) <= gate(xo32, xo), ("inverse vs f64 oracle", rel(xih, xo), rel(xo32, xo))
        if kind == "planar_randn":
            # stress variant: wᵀû → −1 makes log1p(wᵀû·sech²) arbitrarily ill-conditioned near wᵀz + b = 0, so the
            # statistic is a robust (median) one; the gate is still the reference's own error on this input
            med = lambda a: float(np.median(np.abs(a - ljio) / (np.abs(ljio) + 1e-3)))  # noqa: E731
            assert med(ljih) <= max(RTOL, 2 * med(ljio32)), (med(ljih), med(ljio32))
        else:
            lg = gate(ljio32, ljio)
            assert np.linalg.norm(ljih - ljio) <= lg * max(np.linalg.norm(ljio), math.sqrt(N) * 1e-2), (rel(ljih, ljio), lg)
        # inverse∘forward ≈ id: as far from x as the float64 inverse of the device's y is (forward rounding amplified
        # by the inverse's conditioning), plus the inverse's own gate
        assert rel(xih, x) <= rel(xo, x) + gate(xo32, xo), (rel(xih, x), rel(xo, x))


@pytest.mark.parametrize("D", [128, 64, 32, 256, 10])
def test_fused_chain_matches_layerwise_and_oracle(B, D):
    rng = np.random.default_rng(D)
    N = 1537
    # the exp block goes last: exp followed by an affine coupling is ill-conditioned to invert in ANY fp32
    # implementation (the float32 oracle itself loses 1e-2 on such a chain)
    kinds = ["planar", "batchnorm", "radial", "permute", "rqs", "planar", "coupling", "radial", "planar", "stacked"]
    pairs = [make_case(k, D, rng) for k in kinds]
    flow = B.Composed(*[p[0] for p in pairs])
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)
    y, lj = B.with_logabsdet_jacobian(flow, xd)
    yo, ljo = O.chain_forward([p[1] for p in pairs], x.astype(np.float64))
    yo32, ljo32 = O.chain_forward([p[1] for p in pairs], x)
    # 10 chained fp32 layers: the gate is 1e-5 or twice the float32 oracle's own distance to float64
    assert rel(B.to_numpy(y), yo) <= max(RTOL, 2 * rel(yo32, yo)), (rel(B.to_numpy(y), yo), rel(yo32, yo))
    assert rel(B.to_numpy(lj), ljo) <= max(RTOL, 2 * rel(ljo32, ljo)), (rel(B.to_numpy(lj), ljo), rel(ljo32, ljo))
    # the `∘` spelling (outer @ inner) builds the same chain
    comp = pairs[0][0]
    for p in pairs[1:]:
        comp = p[0] @ comp
    y2, lj2 = B.with_logabsdet_jacobian(comp, xd)
    assert np.array_equal(B.to_numpy(y2), B.to_numpy(y)) and np.array_equal(B.to_numpy(lj2), B.to_numpy(lj))
    # layer by layer with the in-place, accumulating variants (with_logabsdet_jacobian!)
    import torch

    buf = xd.t().contiguous().t().clone() if False else B.from_numpy(x)
    acc = torch.zeros(N, dtype=torch.float32, device="cuda")
    for p in pairs:
        buf, acc = B.with_logabsdet_jacobian_(p[0], buf, None, acc)
    assert rel(B.to_numpy(buf), B.to_numpy(y)) <= 2e-6
    assert rel(B.to_numpy(acc), B.to_numpy(lj)) <= 2e-6
    # inverse chain
    xi, lji = B.with_logabsdet_jacobian(B.inverse(flow), y)
    olayers = [p[1] for p in pairs]
    yh = B.to_numpy(y)
    xo, ljio = O.chain_inverse(olayers, yh.astype(np.float64))   # float64 reference on the device's own y
    xo32, ljio32 = O.chain_inverse(olayers, yh)                   # float32 reference on the same y
    assert rel(B.to_numpy(xi), xo) <= gate(xo32, xo), (rel(B.to_numpy(xi), xo), rel(xo32, xo))
    assert rel(B.to_numpy(lji), ljio) <= gate(ljio32, ljio), (rel(B.to_numpy(lji), ljio), rel(ljio32, ljio))
    assert rel(B.to_numpy(xi), x) <= rel(xo, x) + gate(xo32, xo)  # inverse∘forward ≈ id, as well as float64 manages from this y
    # TransformedDistribution logpdf (transformed_distribution.jl:165-169)
    mu, sigma = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 2.0, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu, sigma), flow)
    lp = B.to_numpy(B.logpdf(td, y))
    lpo = O.transformed_logpdf(olayers, mu.astype(np.float64), sigma.astype(np.float64), yh.astype(np.float64))
    lpo32 = O.transformed_logpdf(olayers, mu, sigma, yh)
    assert rel(lp, lpo) <= gate(lpo32, lpo), (rel(lp, lpo), rel(lpo32, lpo))
    tot, lp2 = B.logpdf_sum(td, y)
    assert np.array_equal(B.to_numpy(lp2), lp)
    assert abs(float(tot) - float(lp.astype(np.float64).sum())) <= 1e-9 * abs(float(tot)) + 1e-6


def test_c_abi_single_layer_entry_points(B):
    """Every per-layer symbol of include/b2b.h called directly (plain pointers, no Python layer objects)."""
    import torch

    L = B.lib()
    rng = np.random.default_rng(42)
    D, N = 64, 777
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)
    yd = B.colmajor_empty(D, N)
    ljd = torch.empty(N, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a)).cuda()  # noqa: E731

    def check_pair(fwd, inv, args_dev, olayer, tol=RTOL):
        rc = fwd(xd.data_ptr(), yd.data_ptr(), ljd.data_ptr(), *args_dev, D, N, D, D, 0, s)
        assert rc == 0, L.b2b_status_string(rc)
        yo, ljo = olayer.forward(x.astype(np.float64))
        assert rel(B.to_numpy(yd), yo) <= tol and rel(B.to_numpy(ljd), ljo) <= tol
        # in place inverse: y aliases x
        rc = inv(yd.data_ptr(), yd.data_ptr(), ljd.data_ptr(), *args_dev, D, N, D, D, 1, s)
        assert rc == 0, L.b2b_status_string(rc)
        assert rel(B.to_numpy(yd), x) <= 10 * tol
        assert np.linalg.norm(B.to_numpy(ljd)) <= 1e-4 * math.sqrt(N)  # fwd + inverse logjac cancel

    w, u, b = (rng.standard_normal(D) / 8).astype(f32), (rng.standard_normal(D) / 8).astype(f32), f32([0.2])
    t = [dev(w), dev(u), dev(b)]
    check_pair(L.b2b_planar_fwd_f32, L.b2b_planar_inv_f32, [a.data_ptr() for a in t], O.Layer("planar", dict(w=w, u=u, b=b)))
    a_, be, z0 = f32([0.3]), f32([-0.4]), rng.standard_normal(D).astype(f32)
    t = [dev(a_), dev(be), dev(z0)]
    check_pair(L.b2b_radial_fwd_f32, L.b2b_radial_inv_f32, [a.data_ptr() for a in t], O.Layer("radial", dict(alpha_raw=a_, beta=be, z0=z0)))
    K = 8
    W, H, Dv = O.rqs_params(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    t = [dev(W.T), dev(H.T), dev(Dv.T)]  # Julia column-major (D x K1) == row-major (K1 x D)
    check_pair(L.b2b_rqs_fwd_f32, L.b2b_rqs_inv_f32, [a.data_ptr() for a in t] + [K + 1], O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv)))
    bb, logs, m, v = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    t = [dev(bb), dev(logs), dev(m), dev(v)]
    check_pair(L.b2b_batchnorm_eval_fwd_f32, L.b2b_batchnorm_eval_inv_f32, [a.data_ptr() for a in t] + [1e-5],
               O.Layer("batchnorm", dict(bn=O.BatchNormParams(bb, logs, m, v, f32(1e-5), f32(0.1)))))
    n1 = D // 2
    idx1, idx2 = np.arange(n1, dtype=np.int32), np.arange(n1, D, dtype=np.int32)
    Wc, c = (rng.standard_normal((2 * n1, D - n1)) * 0.05).astype(f32), (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    t = [dev(idx1), dev(idx2), dev(Wc.T), dev(c)]
    args = [t[0].data_ptr(), n1, -1, t[1].data_ptr(), D - n1, -1, t[2].data_ptr(), t[3].data_ptr()]
    # the coupling entry points take (workspace, bytes) before the stream: NULL workspace = fp32 CUDA-core kernel
    cf = lambda *a: L.b2b_coupling_affine_fwd_f32(*a[:-1], None, 0, a[-1])  # noqa: E731
    ci = lambda *a: L.b2b_coupling_affine_inv_f32(*a[:-1], None, 0, a[-1])  # noqa: E731
    check_pair(cf, ci, args, O.Layer("coupling_affine", dict(idx1=idx1 + 1, idx2=idx2 + 1, W=Wc, c=c)))
    # permute + stacked + mvnormal
    perm = rng.permutation(D).astype(np.int32)
    pd = dev(perm)
    assert L.b2b_permute_rows_f32(xd.data_ptr(), yd.data_ptr(), ljd.data_ptr(), pd.data_ptr(), 0, D, N, D, D, 0, s) == 0
    ye = np.empty_like(x)
    ye[perm] = x
    assert np.array_equal(B.to_numpy(yd), ye) and np.all(B.to_numpy(ljd) == 0)
    assert L.b2b_permute_rows_f32(yd.data_ptr(), yd.data_ptr(), None, pd.data_ptr(), 1, D, N, D, D, 0, s) == 0
    assert np.array_equal(B.to_numpy(yd), x)
    code = np.zeros(D, np.int32)
    code[:4] = 1
    code[4:8] = 2
    av = np.zeros(D, f32)
    xp = np.abs(x) + f32(0.1)
    xpd = B.from_numpy(xp)
    cd, ad = dev(code), dev(av)
    assert L.b2b_stacked_elementwise_f32(xpd.data_ptr(), yd.data_ptr(), ljd.data_ptr(), cd.data_ptr(), ad.data_ptr(), None, 0, D, N, D, D, 0, s) == 0
    ye = xp.copy()
    ye[:4] = np.exp(xp[:4])
    ye[4:8] = np.log(xp[4:8])
    assert rel(B.to_numpy(yd), ye) <= 1e-6
    assert rel(B.to_numpy(ljd), xp[:4].sum(0) - np.log(xp[4:8]).sum(0)) <= 1e-5
    mu, sg = rng.standard_normal(D).astype(f32), rng.uniform(0.5, 2, D).astype(f32)
    mud, sgd = dev(mu), dev(sg)
    lj_in = rng.standard_normal(N).astype(f32)
    ljin_d = dev(lj_in)
    out = torch.empty(N, device="cuda")
    sm = torch.zeros((), dtype=torch.float64, device="cuda")
    ws = torch.empty(4096 * 8, dtype=torch.uint8, device="cuda")
    rc = L.b2b_mvnormal_diag_logpdf_f32(xd.data_ptr(), mud.data_ptr(), sgd.data_ptr(), ljin_d.data_ptr(), out.data_ptr(),
                                        sm.data_ptr(), D, N, D, ws.data_ptr(), ws.numel(), s)
    assert rc == 0, L.b2b_status_string(rc)
    ref = O.mvnormal_diag_logpdf(mu.astype(np.float64), sg.astype(np.float64), x.astype(np.float64)) + lj_in
    assert rel(B.to_numpy(out), ref) <= RTOL
    assert abs(float(sm) - ref.sum()) <= 1e-5 * abs(ref.sum())
    # error convention: negative status, never a crash
    assert L.b2b_planar_fwd_f32(None, yd.data_ptr(), ljd.data_ptr(), None, None, None, D, N, D, D, 0, s) == -1
    assert L.b2b_rqs_fwd_f32(xd.data_ptr(), yd.data_ptr(), ljd.data_ptr(), t[0].data_ptr(), t[0].data_ptr(), t[0].data_ptr(), 1, D, N, D, D, 0, s) == -1
    assert b"invalid" in L.b2b_status_string(-1)


def test_reference_golden_vectors_on_device(B, golden):
    import torch

    # Permute (test/bijectors/permute.jl:30-64) incl. the 4 constructor spellings; bit-exact payloads
    g = golden["permute_3"]
    bs = [B.Permute(np.array(g["matrix"])), B.Permute(g["indices"]), B.Permute(3, *[tuple(p) for p in g["pairs"]]),
          B.Permute(3, *[(p[0], p[1]) for p in g["vector_pairs"]])]
    assert all(b == bs[0] for b in bs)
    x = B.from_numpy(np.array(g["x"], f32))
    for b in bs:
        y, lj = B.with_logabsdet_jacobian(b, x)
        assert B.to_numpy(y).tolist() == g["y"] and float(lj) == 0.0
        assert B.to_numpy(B.inverse(b)(b(x))).tolist() == g["x"]
    for case in golden["permute_invalid"]["cases"]:
        with pytest.raises(ValueError):
            if "pairs" in case:
                B.Permute(case["n"], *[tuple(p) for p in case["pairs"]])
            else:
                B.Permute(case["n"], *[(p[0], p[1]) for p in case["vector_pairs"]])
    payload = np.array([np.nan, -0.0, 1.5, np.inf], dtype=f32)
    payload.view(np.uint32)[0] = 0x7FC12345  # NaN with a payload
    yb = B.to_numpy(B.Permute([3, 1, 4, 2])(B.from_numpy(payload)))
    assert yb.view(np.uint32).tolist() == payload.view(np.uint32)[[1, 3, 0, 2]].tolist()
    # Coupling with the Shift law x₁ + x₂ (test/bijectors/coupling.jl:18-42) as s = 0, t = x₂
    g = golden["coupling_shift"]
    cl = B.Coupling(B.AffineConditioner(np.array([[0.0], [1.0]], f32)), B.PartitionMask(3, [1], [2]))
    x = B.from_numpy(np.array(g["x"], f32))
    y, lj = B.with_logabsdet_jacobian(cl, x)
    assert B.to_numpy(y).tolist() == g["y"] and float(lj) == 0.0
    xi, lji = B.with_logabsdet_jacobian(B.inverse(cl), y)
    assert B.to_numpy(xi).tolist() == g["x"] and float(lji) == 0.0
    m = B.PartitionMask(3, [1], [2])
    assert m == B.PartitionMask(3, [1], [2], [3]) and m.indices_3 == [3]
    # Planar deterministic case (test/normalising_flows.jl:37-42)
    flow = B.PlanarLayer(np.ones(10, f32), np.zeros(10, f32), f32(1.0))
    z = B.from_numpy(np.ones((10, 100), f32))
    y, lj = B.with_logabsdet_jacobian(flow, z)
    uh = (math.log(2) - 1) / 10
    assert rel(B.to_numpy(y), np.full((10, 100), 1 + uh * math.tanh(11.0))) <= 1e-6
    assert np.allclose(B.to_numpy(lj), math.log1p((math.log(2) - 1) / math.cosh(11.0) ** 2), rtol=1e-4, atol=1e-12)
    assert rel(B.to_numpy(B.inverse(flow)(flow(z))), np.ones((10, 100))) <= 1e-6
    # Radial deterministic case (test/normalising_flows.jl:86-91): β̂ = 0 ⇒ identity
    rflow = B.RadialLayer(f32(1.0), f32(1.0), np.zeros(10, f32))
    y, lj = B.with_logabsdet_jacobian(rflow, z)
    assert rel(B.to_numpy(y), np.ones((10, 100))) <= 1e-6 and np.abs(B.to_numpy(lj)).max() <= 1e-5
    assert rel(B.to_numpy(B.inverse(rflow)(rflow(z))), np.ones((10, 100))) <= 1e-6
    # InvertibleBatchNorm defaults (test/normalising_flows.jl:7-23)
    bn = B.InvertibleBatchNorm(2)
    xr = np.random.default_rng(1).standard_normal((2, 20)).astype(f32)
    xd = B.from_numpy(xr)
    y, lj = B.with_logabsdet_jacobian(bn, xd)
    assert rel(B.to_numpy(y), xr / np.sqrt(f32(1) + f32(1e-5))) <= 1e-6
    assert np.allclose(B.to_numpy(lj), -math.log(1 + 1e-5), rtol=1e-2)
    assert rel(B.to_numpy(B.inverse(bn)(bn(xd))), xr) <= 1e-6
    assert B.inverse(B.inverse(bn)) == bn
    with pytest.raises(RuntimeError, match="expected 2 channels"):
        B.with_logabsdet_jacobian(bn, B.from_numpy(np.zeros((10, 2), f32)))
    # RQS outside the box is the identity with zero logjac (test/bijectors/rational_quadratic_spline.jl:47-61)
    rng = np.random.default_rng(5)
    b_mv = B.RationalQuadraticSpline(rng.standard_normal((2, 3)), rng.standard_normal((2, 3)), rng.standard_normal((2, 2)), 2)
    xo = B.from_numpy(np.array([-5.0, 5.0], f32))
    y, lj = B.with_logabsdet_jacobian(b_mv, xo)
    assert B.to_numpy(y).tolist() == [-5.0, 5.0] and float(lj) == 0.0
    W, H, Dv = b_mv.knots()
    assert np.allclose(W[:, 0], -2) and np.allclose(W[:, -1], 2, rtol=1e-6) and np.all(Dv[:, 0] == 1) and np.all(Dv[:, -1] == 1)
    with pytest.raises(AssertionError):
        B.RationalQuadraticSpline(W, H, -Dv)
    # Stacked value test (test/bijectors/stacked.jl:100-108)
    sb = B.Stacked([B.elementwise("exp"), B.elementwise("log"), B.Shift(5.0)])
    y, lj = B.with_logabsdet_jacobian(sb, B.from_numpy(np.ones(3, f32)))
    assert np.allclose(B.to_numpy(y), [math.e, 0.0, 6.0], rtol=1e-6) and float(lj) == pytest.approx(1.0, rel=1e-6)
    with pytest.raises(RuntimeError, match="input length mismatch"):
        sb(B.from_numpy(np.ones(4, f32)))
    # elementwise(exp) doctest (src/interface.jl:21-31) -- host plumbing, Float64
    ye, le = B.with_logabsdet_jacobian(B.elementwise("exp"), torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64))
    assert ye.tolist() == golden["elementwise_exp_doctest"]["y"] and float(le) == 6.0


def test_find_alpha_residual_on_device(B, golden):
    """test/normalising_flows.jl:47-71 restated for the fp32 device solver through a D=1 PlanarLayer
    (w = 1 ⇒ û = wᵀû = softplus(u) − 1, and inverse(y) IS α)."""
    g = golden["find_alpha_grid"]
    for c in g["wt_u_hat"]:
        if c <= -1.0:
            continue  # c = −1 needs u = −∞
        u = math.log(math.expm1(c + 1.0)) if c + 1.0 < 30 else c + 1.0
        for b in g["b"]:
            flow = B.PlanarLayer(np.ones(1, f32), f32([u]), f32([b]))
            ys = np.array(g["wt_y"], f32)[None, :]
            alpha = B.to_numpy(B.inverse(flow)(B.from_numpy(ys))).astype(np.float64)[0]
            c32 = float(np.log1p(np.exp(np.float64(f32(u)))) - 1.0)
            resid = alpha + c32 * np.tanh(alpha + float(f32(b))) - ys[0].astype(np.float64)
            # What comes back is z = y − û·tanh(α+b) (planar_layer.jl:124), not α itself: the fp32 quantisation of
            # α (½ ulp) is amplified by û·sech² into z and again by f′ = 1 + c·sech² into the residual, so the
            # fp32 floor is ~eps·(1+|c|)²·(|y|+|c|+1).  (The reference checks α in Float64 with rtol = sqrt(eps).)
            eps32 = float(np.finfo(np.float32).eps)
            tol = 4 * eps32 * (1 + abs(c32)) ** 2 * (np.abs(ys[0]) + abs(c32) + 1.0)
            assert np.all(np.abs(resid) <= tol), (c, b, resid, tol)
    # issue 204 (b = −1e8): α ≈ wt_y + wt_u_hat
    gi = golden["find_alpha_issue_204"]
    u = math.log(math.expm1(gi["wt_u_hat"] + 1.0))
    flow = B.PlanarLayer(np.ones(1, f32), f32([u]), f32([gi["b"]]))
    a = float(B.to_numpy(B.inverse(flow)(B.from_numpy(np.array([gi["wt_y"]], f32))))[0])
    assert a == pytest.approx(gi["wt_y"] + gi["wt_u_hat"], rel=1e-5)


F64_KINDS = ["planar", "planar_randn", "radial", "rqs", "batchnorm", "permute", "coupling", "stacked", "leaky_relu", "bounded"]


def make_case64(kind, D, rng):
    """(Float64 device layer, oracle layer): the Float32 cases rebuilt with Float64 parameters."""
    import torch

    import bijectors_jl_b200 as B

    f64 = torch.float64
    lay, olay = make_case(kind, D, rng)
    p = olay.params
    if kind in ("planar", "planar_randn"):
        w, u, b = (p[k].astype(np.float64) + 1e-9 * rng.standard_normal(p[k].shape) for k in ("w", "u", "b"))  # not fp32-representable
        return B.PlanarLayer(w, u, b, dtype=f64), O.Layer("planar", dict(w=w, u=u, b=b))
    if kind == "radial":
        a, be, z0 = (p[k].astype(np.float64) + 1e-9 * rng.standard_normal(p[k].shape) for k in ("alpha_raw", "beta", "z0"))
        return B.RadialLayer(a, be, z0, dtype=f64), O.Layer("radial", dict(alpha_raw=a, beta=be, z0=z0))
    if kind == "rqs":
        K = 8
        rw, rh, rd = rng.standard_normal((D, K)), rng.standard_normal((D, K)), rng.standard_normal((D, K - 1))
        l64 = B.RationalQuadraticSpline(rw, rh, rd, 3.0, dtype=f64)
        W, H, Dv = l64.knots()
        assert W.dtype == np.float64
        return l64, O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv))
    if kind == "batchnorm":
        bn = p["bn"]
        b, logs, m, v = (np.asarray(t, np.float64) + 1e-9 * rng.standard_normal(D) for t in (bn.b, bn.logs, bn.m, bn.v))
        return (B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v, dtype=f64),
                O.Layer("batchnorm", dict(bn=O.BatchNormParams(b, logs, m, v, np.float64(np.float32(1e-5)), np.float64(0.1)))))
    if kind == "coupling":
        W, c = p["W"].astype(np.float64) + 1e-9 * rng.standard_normal(p["W"].shape), p["c"].astype(np.float64)
        return (B.Coupling(B.AffineConditioner(W, c, dtype=f64), B.PartitionMask(D, list(p["idx1"]), list(p["idx2"]))),
                O.Layer("coupling_affine", dict(idx1=p["idx1"], idx2=p["idx2"], W=W, c=c)))
    if kind in ("stacked", "leaky_relu", "bounded"):
        # the scalar law parameters are Python floats on the device side: give the oracle the same float64 values (the
        # Float32 cases carry float32-rounded constants)
        ops = [tuple([op[0]] + [{-1.7: -1.7, 0.3: 0.3, 0.1: 0.1}.get(round(float(v), 6), float(v)) for v in op[1:]]) for op in p["ops"]]
        return (B.Stacked(lay.bs, lay.ranges_in, dtype=f64) if hasattr(lay, "bs") else lay), O.Layer("stacked", dict(ops=ops, ranges=p["ranges"]))
    return lay, olay  # permute: no floating-point parameters


@pytest.mark.parametrize("D,N", [(128, 300), (32, 257), (10, 100), (3, 7), (200, 33)])
@pytest.mark.parametrize("kind", F64_KINDS)
def test_float64_layers_match_the_float64_oracle(B, kind, D, N):
    """Float64 batches with Float64 parameters (b2b_chain_run_f64): the reference is generic in its element type and its
    own tests run in Float64.  Against the float64 oracle the gate is 1e-12 relative (ill-conditioned planar_randn: 1e-9),
    bit-exact for Permute."""
    if kind in ("coupling", "stacked", "bounded") and D < 3:
        pytest.skip("needs D >= 3")
    import zlib

    rng = np.random.default_rng(zlib.crc32(f"f64-{kind}-{D}-{N}".encode()))
    lay, olay = make_case64(kind, D, rng)
    x = rng.standard_normal((D, N)) * (1.5 if kind == "rqs" else 1.0)
    if kind == "bounded":
        x = rng.uniform(-0.9, 2.9, (D, N))
    xd = B.from_numpy(x, dtype=np.float64)
    y, lj = B.with_logabsdet_jacobian(lay, xd)
    assert y.dtype == lj.dtype and str(y.dtype) == "torch.float64"
    yo, ljo = olay.forward(x)
    yh, ljh = B.to_numpy(y), B.to_numpy(lj)
    tol = 1e-9 if kind == "planar_randn" else 1e-12
    if kind == "permute":
        assert np.array_equal(yh.view(np.uint64), yo.view(np.uint64)) and np.all(ljh == 0)
    else:
        assert rel(yh, yo) <= tol, rel(yh, yo)
        assert np.linalg.norm(ljh - ljo) <= tol * max(np.linalg.norm(ljo), math.sqrt(N) * 1e-2), rel(ljh, ljo)
    xi, lji = B.with_logabsdet_jacobian(B.inverse(lay), y)
    xo, ljio = olay.inverse(yh)
    if kind == "permute":
        assert np.array_equal(B.to_numpy(xi).view(np.uint64), x.view(np.uint64))
    else:
        assert rel(B.to_numpy(xi), xo) <= (1e-7 if kind == "planar_randn" else 1e-11), rel(B.to_numpy(xi), xo)
        if kind != "planar_randn":
            assert np.linalg.norm(B.to_numpy(lji) - ljio) <= 1e-10 * max(np.linalg.norm(ljio), math.sqrt(N) * 1e-2)
    # the Float32 layers refuse a Float64 batch (and vice versa) instead of silently converting
    if kind == "planar":
        with pytest.raises(TypeError):
            B.with_logabsdet_jacobian(make_case(kind, D, rng)[0], xd)


def test_float64_chain_logpdf_and_find_alpha_grid(B, golden):
    """A heterogeneous Float64 chain + TransformedDistribution logpdf + batch sum against the float64 oracle, and the
    reference's find_alpha test in ITS precision: residual grid with atol = 1e-14 where wt_y = 0, issue 204
    (test/normalising_flows.jl:47-71)."""
    import torch

    f64 = torch.float64
    rng = np.random.default_rng(64)
    D, N = 64, 501
    kinds = ["planar", "batchnorm", "radial", "permute", "rqs", "coupling", "planar", "stacked"]
    pairs = [make_case64(k, D, rng) for k in kinds]
    flow = B.Composed(*[p[0] for p in pairs])
    olayers = [p[1] for p in pairs]
    x = rng.standard_normal((D, N))
    y, lj = B.with_logabsdet_jacobian(flow, B.from_numpy(x, dtype=np.float64))
    yo, ljo = O.chain_forward(olayers, x)
    assert rel(B.to_numpy(y), yo) <= 1e-12 and rel(B.to_numpy(lj), ljo) <= 1e-12, (rel(B.to_numpy(y), yo), rel(B.to_numpy(lj), ljo))
    mu, sigma = rng.standard_normal(D) * 0.1, rng.uniform(0.5, 2.0, D)
    td = B.transformed(B.MvNormal(D, mu, sigma, dtype=f64), flow)
    tot, lp = B.logpdf_sum(td, y)
    lpo = O.transformed_logpdf(olayers, mu, sigma, B.to_numpy(y))
    assert rel(B.to_numpy(lp), lpo) <= 1e-10, rel(B.to_numpy(lp), lpo)
    assert abs(float(tot) - float(lpo.sum())) <= 1e-10 * abs(float(lpo.sum()))
    # find_alpha through a D = 1 PlanarLayer with w = 1: inverse(y) = y − û·tanh(α+b) and wᵀû = softplus(u) − 1
    g = golden["find_alpha_grid"]
    for c in g["wt_u_hat"]:
        if c <= -1.0:
            continue  # c = −1 needs u = −∞
        u = math.log(math.expm1(c + 1.0)) if c + 1.0 < 30 else c + 1.0
        cc = math.log1p(math.exp(u)) - 1.0 if u < 30 else u - 1.0
        for b in g["b"]:
            lay = B.PlanarLayer(np.ones(1), np.array([u]), np.array([b]), dtype=f64)
            ys = np.array(g["wt_y"], np.float64)[None, :]
            # with w = 1: û = wᵀû = cc and z = y − û·tanh(α+b) = α, so the inverse's output IS the root
            alpha = B.to_numpy(B.inverse(lay)(B.from_numpy(ys, dtype=np.float64)))[0]
            rhs = alpha + cc * np.tanh(alpha + b)
            # the reference's check: wt_y ≈ α + wt_u_hat·tanh(α + b) (rtol = sqrt(eps)), atol = 1e-14 when wt_y == 0;
            # here 1e-12 relative (z is rebuilt from the root: ½ ulp of α is amplified by f′ = 1 + c·sech² <= 1 + |c|)
            for yv, rv in zip(ys[0], rhs):
                if yv == 0.0:
                    assert abs(rv) <= 1e-14 * (1 + abs(cc)) ** 2, (c, b, rv)
                else:
                    assert abs(rv - yv) <= 1e-12 * max(abs(rv), abs(yv)) * (1 + abs(cc)), (c, b, yv, rv)
    gi = golden["find_alpha_issue_204"]
    u = math.log(math.expm1(gi["wt_u_hat"] + 1.0))
    lay = B.PlanarLayer(np.ones(1), np.array([u]), np.array([gi["b"]]), dtype=f64)
    z = float(B.to_numpy(B.inverse(lay)(B.from_numpy(np.array([[gi["wt_y"]]]), dtype=np.float64)))[0, 0])
    # b = −1e8: tanh(α + b) = −1, so z = y + wᵀû and α = wt_y + wt_u_hat (planar_layer.jl issue 204)
    assert z == pytest.approx(gi["wt_y"] + gi["wt_u_hat"], rel=1e-14)


def test_host_buffer_entry_point_matches_device_path(B):
    import torch

    rng = np.random.default_rng(8)
    D, N = 128, 200_000  # > 3 chunks of 2^16 columns: exercises the multi-stream pipeline and the tail
    pairs = [make_case("planar", D, rng) for _ in range(4)]
    flow = B.Composed(*[p[0] for p in pairs])
    xh = B.from_numpy(rng.standard_normal((D, N)).astype(f32), device="cpu", pin_memory=True)
    yh, ljh = B.with_logabsdet_jacobian(flow, xh)
    assert not yh.is_cuda and yh.is_pinned()
    yd, ljd = B.with_logabsdet_jacobian(flow, xh.cuda())
    assert np.array_equal(B.to_numpy(yh), B.to_numpy(yd)) and np.array_equal(B.to_numpy(ljh), B.to_numpy(ljd))
    td = B.transformed(B.MvNormal(D), flow)
    tot_h, lp_h = B.logpdf_sum(td, yh)
    tot_d, lp_d = B.logpdf_sum(td, yd)
    assert np.array_equal(B.to_numpy(lp_h), B.to_numpy(lp_d))
    assert abs(float(tot_h) - float(tot_d)) <= 1e-9 * abs(float(tot_d))


def test_full_size_properties_config2(B):
    """BASELINE config 2 at FULL size (8×Planar, D=128, N=2^20): size-independent properties + a
    4096-column sample against the oracle."""
    import torch

    rng = np.random.default_rng(100)
    D, N, Lc = 128, 1 << 20, 8
    pairs = [make_case("planar", D, np.random.default_rng(100 + l)) for l in range(Lc)]
    flow = B.Composed(*[p[0] for p in pairs])
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((N, D), device="cuda", generator=gen).t()
    y, lj = B.with_logabsdet_jacobian(flow, x)
    assert y.shape == (D, N) and lj.shape == (N,) and bool(torch.isfinite(y).all()) and bool(torch.isfinite(lj).all())
    cols = np.sort(rng.choice(N, 4096, replace=False))
    ct = torch.as_tensor(cols, device="cuda")
    xs = x[:, ct].cpu().numpy()
    yo, ljo = O.chain_forward([p[1] for p in pairs], xs.astype(np.float64))
    assert rel(y[:, ct].cpu().numpy(), yo) <= RTOL and rel(lj[ct].cpu().numpy(), ljo) <= RTOL
    xi, lji = B.with_logabsdet_jacobian(B.inverse(flow), y)
    olayers = [p[1] for p in pairs]
    ys = y[:, ct].cpu().numpy()
    xo, ljio = O.chain_inverse(olayers, ys.astype(np.float64))  # inverse OUTPUTS against the oracle on the sample
    xo32, ljio32 = O.chain_inverse(olayers, ys)
    gx, gl = gate(xo32, xo), gate(ljio32, ljio)
    assert rel(xi[:, ct].cpu().numpy(), xo) <= gx and rel(lji[ct].cpu().numpy(), ljio) <= gl, (rel(xi[:, ct].cpu().numpy(), xo), gx, rel(lji[ct].cpu().numpy(), ljio), gl)
    rt_x, rt_l = 2 * (rel(xo, xs) + gx), 2 * (rel(ljio, -ljo) + gl)
    assert rt_x <= 1e-4 and rt_l <= 1e-4, (rt_x, rt_l)
    assert float((xi - x).norm() / x.norm()) <= rt_x  # inverse∘forward ≈ id
    assert float((lji + lj).norm()) <= rt_l * max(float(lj.norm()), 1.0)  # ires == (x, −logjac)
    # column independence: a permuted batch gives permuted outputs (bit-identical)
    perm = torch.randperm(N, device="cuda")[: 1 << 16]
    y2, lj2 = B.with_logabsdet_jacobian(flow, x[:, perm].t().contiguous().t())
    assert torch.equal(y2, y[:, perm]) and torch.equal(lj2, lj[perm])
    # variant cross-check: every kernel variant gives the same answer as the v0 kernel
    B.lib().b2b_set_kernel_variant(1)
    try:
        y0, lj0 = B.with_logabsdet_jacobian(flow, x)
    finally:
        B.lib().b2b_set_kernel_variant(0)
    assert float((y0 - y).norm() / y.norm()) <= 2e-6 and float((lj0 - lj).norm() / lj.norm()) <= 2e-6


@pytest.mark.parametrize("D", [128, 64, 32, 256, 10, 7])
def test_rand_matches_the_oracle_stream(B, D):
    """rand(td, n) with the base samples generated inside the chain kernel (Philox4x32-10 + Box-Muller): the samples
    equal the oracle's restatement of the stream pushed through the oracle's chain (fixed seed = fixed base sample),
    a column shard continues the global stream, and the result does not depend on which kernel draws them."""
    rng = np.random.default_rng(50 + D)
    n = 2300
    seed, off = 0x1234_5678_9ABC_DEF0, 5
    mu, sigma = (rng.standard_normal(D) * 0.3).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    base = B.MvNormal(D, mu, sigma)
    zo = O.philox_normals(seed, off, D, n, mu=mu.astype(np.float64), sigma=sigma.astype(np.float64))
    z = B.to_numpy(base.rand(n, seed=seed, offset=off))
    assert z.shape == (D, n) and rel(z, zo) <= 3e-6, rel(z, zo)  # MUFU sin/cos/lg2: ~2^-21 absolute
    assert np.array_equal(B.to_numpy(base.rand(n, seed=seed, offset=off)), z)            # deterministic
    assert np.array_equal(B.to_numpy(base.rand(500, seed=seed, offset=off, column_offset=700)), z[:, 700:1200])
    assert not np.array_equal(B.to_numpy(base.rand(n, seed=seed + 1, offset=off)), z)
    kinds = ["planar", "radial", "batchnorm", "planar"] if D not in (10, 7) else ["planar", "radial"]
    pairs = [make_case(k, D, rng) for k in kinds]
    td = B.transformed(base, B.Composed(*[p[0] for p in pairs]))
    y, lj = B.rand(td, n, seed=seed, offset=off, with_logjac=True)
    yo, ljo = O.chain_forward([p[1] for p in pairs], zo)
    assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL, (rel(B.to_numpy(y), yo), rel(B.to_numpy(lj), ljo))
    # the fused sampler and "base samples, then the chain" are the same computation
    y2, lj2 = B.with_logabsdet_jacobian(td.transform, B.from_numpy(z))
    assert rel(B.to_numpy(y), B.to_numpy(y2)) <= 2e-6 and rel(B.to_numpy(lj), B.to_numpy(lj2)) <= 2e-6
    # logpdf of the samples is the base density minus the log-Jacobian (test/normalising_flows.jl:97-111)
    lp = B.to_numpy(B.logpdf(td, y))
    olayers, yh = [p[1] for p in pairs], B.to_numpy(y)
    lpo = O.transformed_logpdf(olayers, mu.astype(np.float64), sigma.astype(np.float64), yh.astype(np.float64))
    assert rel(lp, lpo) <= gate(O.transformed_logpdf(olayers, mu, sigma, yh), lpo)
    lps = O.mvnormal_diag_logpdf(mu.astype(np.float64), sigma.astype(np.float64), zo) - ljo  # density of the sample itself
    assert rel(lpo, lps) <= 1e-4  # (what the float32 rounding of y costs the float64 oracle)


def test_rand_and_shapes(B):
    import torch

    rng = np.random.default_rng(3)
    D = 64
    flow = B.Composed(*[make_case("radial", D, rng)[0] for _ in range(3)])
    td = B.transformed(B.MvNormal(D), flow)
    s = B.rand(td, 1000, seed=0)
    assert s.shape == (D, 1000) and s.stride(0) == 1 and bool(torch.isfinite(s).all())
    lp = B.logpdf(td, s)
    assert lp.shape == (1000,) and bool(torch.isfinite(lp).all())
    assert not B.isclosedform(B.inverse(B.PlanarLayer(4))) and B.isclosedform(flow)


_TC_SHORT = 64 * 37 + 29  # at most one 64-column tile per CTA
_TC_LONG = 64 * 132 * 9 + 29  # nine tiles per CTA on 132 SMs: the stage barriers and the column-scale ring wrap
_TC_CASES = [(256, 128, 0, 128, 128, _TC_SHORT), (256, 128, 128, 128, 0, _TC_SHORT), (128, 64, 0, 64, 64, _TC_SHORT),
             (256, 64, 0, 128, 128, _TC_SHORT), (192, 100, 64, 64, 0, _TC_SHORT), (256, 128, 0, 128, 128, _TC_LONG)]


@pytest.mark.parametrize("D,n1,row1,n2,row2,N", _TC_CASES,
                         ids=["-".join(map(str, c[:5])) + ("" if c[5] == _TC_SHORT else "-many_tiles") for c in _TC_CASES])
def test_coupling_tensor_core_path(B, D, n1, row1, n2, row2, N):
    """The wgmma path (fp16 hi/lo split, 3 products, fp32 register accumulation) against the oracle and against the
    exact-fp32 CUDA-core kernel; masks with pass-through rows (x₃), out-of-place, in-place, N tail."""
    import torch

    rng = np.random.default_rng(D + n1 + row1)
    idx1 = list(range(row1 + 1, row1 + n1 + 1))
    idx2 = list(range(row2 + 1, row2 + n2 + 1))
    W = (rng.standard_normal((2 * n1, n2)) * 0.3 / np.sqrt(n2)).astype(f32)
    c = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    cl = B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2))
    ol = O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c))
    # every column has its own magnitude (exercises the per-column power-of-two operand scaling)
    x = (rng.standard_normal((D, N)) * np.exp(0.7 * rng.standard_normal(N))[None, :]).astype(f32)
    x[:, 5] *= 1e-20  # tiny / huge / all-zero columns must survive the rescale
    x[:, 6] *= 1e4
    x[:, 7] = 0.0
    xd = B.from_numpy(x)
    y, lj = B.with_logabsdet_jacobian(cl, xd)
    launches = B.lib().b2b_last_launch_count()
    # W preparation + tensor-core kernel on the whole 64-column tiles + the exact-fp32 kernel on the ragged tail
    assert launches == 3, "tensor-core path not taken (W preparation + main kernel + ragged-tail kernel expected)"
    yo, ljo = ol.forward(x.astype(np.float64))
    yo32, ljo32 = ol.forward(x)
    ok = np.isfinite(yo).all(axis=0) & np.isfinite(B.to_numpy(y)).all(axis=0)  # exp overflow in the 1e4 column is legit
    assert ok.sum() >= N - 1
    assert rel(B.to_numpy(y)[:, ok], yo[:, ok]) <= RTOL, rel(B.to_numpy(y)[:, ok], yo[:, ok])
    assert rel(B.to_numpy(lj), ljo) <= RTOL
    B.lib().b2b_set_kernel_variant(10)  # force the exact-fp32 CUDA-core kernel
    try:
        y2, lj2 = B.with_logabsdet_jacobian(cl, xd)
        assert B.lib().b2b_last_launch_count() == 1
    finally:
        B.lib().b2b_set_kernel_variant(0)
    # both kernels carry independent fp32-level noise: each is within 1e-5 of float64, so within 2e-5 of each other
    assert rel(B.to_numpy(y)[:, ok], B.to_numpy(y2)[:, ok]) <= 2e-5 and rel(B.to_numpy(lj), B.to_numpy(lj2)) <= 2e-5
    # the tensor-core result is at least as close to float64 as the float32 reference restatement is (x2 slack)
    assert rel(B.to_numpy(y)[:, ok], yo[:, ok]) <= max(2 * rel(yo32[:, ok], yo[:, ok]), 2e-6)
    # pass-through rows are bit-identical
    keep = np.setdiff1d(np.arange(D), np.asarray(idx1) - 1)
    assert np.array_equal(B.to_numpy(y)[keep], x[keep])
    # inverse (against the float64 oracle applied to the SAME float32 y), in place, accumulating the log-Jacobian
    yh = B.to_numpy(y).copy()
    xo, ljio = ol.inverse(yh[:, ok].astype(np.float64))
    # the many-tile batch draws columns with s down to about -17, where y₁ − t cancels and exp(−s) amplifies it: there the
    # float32 restatement of the reference is itself ~2e-3 away from float64, so that case is held to gate()
    tol = RTOL if N == _TC_SHORT else gate(ol.inverse(yh[:, ok])[0], xo)
    acc = lj.clone()
    yi, acc = B.with_logabsdet_jacobian_(B.inverse(cl), y, None, acc)
    assert yi.data_ptr() == y.data_ptr()
    assert rel(B.to_numpy(yi)[:, ok], xo) <= tol, (rel(B.to_numpy(yi)[:, ok], xo), tol)
    assert float(acc[torch.as_tensor(ok, device="cuda")].abs().max()) <= 1e-4 * max(1.0, float(np.abs(ljo).max()))
    # logabsdetjac alone (no D x N store)
    assert rel(B.to_numpy(B.logabsdetjac(cl, xd)), ljo) <= RTOL


def test_realnvp_config5_shape(B):
    """BASELINE config 5 per-GPU shape: 4 x (affine Coupling + InvertibleBatchNorm), D = 256, alternating masks,
    TransformedDistribution(MvNormal) logpdf -- at a reduced N against the oracle, and the batch sum."""
    rng = np.random.default_rng(400)
    D, N = 256, 1 << 14
    dev_layers, ora_layers = [], []
    for l in range(4):
        first = l % 2 == 0
        idx1 = list(range(1, 129)) if first else list(range(129, 257))
        idx2 = list(range(129, 257)) if first else list(range(1, 129))
        W = (rng.standard_normal((256, 128)) * 0.05 / np.sqrt(128)).astype(f32)
        c = np.zeros(256, f32)
        dev_layers.append(B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2)))
        ora_layers.append(O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c)))
        b, logs, m = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
        v = rng.uniform(0.5, 1.5, D).astype(f32)
        dev_layers.append(B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v))
        ora_layers.append(O.Layer("batchnorm", dict(bn=O.BatchNormParams(b, logs, m, v, f32(1e-5), f32(0.1)))))
    flow = B.Composed(*dev_layers)
    td = B.transformed(B.MvNormal(D), flow)
    yv = rng.standard_normal((D, N)).astype(f32)
    yd = B.from_numpy(yv)
    lp = B.to_numpy(B.logpdf(td, yd))
    lpo = O.transformed_logpdf(ora_layers, None, None, yv.astype(np.float64))
    assert rel(lp, lpo) <= RTOL, rel(lp, lpo)
    tot, lp2 = B.logpdf_sum(td, yd)
    assert abs(float(tot) - lpo.sum()) <= 1e-5 * abs(lpo.sum())
    xs, ljf = B.with_logabsdet_jacobian(flow, yd)
    n_folded = B.lib().b2b_last_launch_count()
    xo, ljo = O.chain_forward(ora_layers, yv.astype(np.float64))
    assert rel(B.to_numpy(xs), xo) <= RTOL and rel(B.to_numpy(ljf), ljo) <= RTOL
    # BatchNorm layers ride inside the coupling launches: 4 x (fold table + W image + wgmma kernel), no BN launch
    assert n_folded == 12, n_folded
    B.lib().b2b_set_kernel_variant(100)  # same chain with the BatchNorm layers as their own launches
    try:
        xs2, ljf2 = B.with_logabsdet_jacobian(flow, yd)
        assert B.lib().b2b_last_launch_count() == 12  # 4 x (W image + kernel) + 4 BatchNorm launches
        lp3 = B.to_numpy(B.logpdf(td, yd))
    finally:
        B.lib().b2b_set_kernel_variant(0)
    assert rel(B.to_numpy(xs), B.to_numpy(xs2)) <= 2e-6 and rel(B.to_numpy(ljf), B.to_numpy(ljf2)) <= 2e-6
    assert rel(lp, lp3) <= 2e-6
    # the fp32 CUDA-core coupling kernel folds BatchNorm the same way
    B.lib().b2b_set_kernel_variant(10)
    try:
        xs3, ljf3 = B.with_logabsdet_jacobian(flow, yd)
        assert B.lib().b2b_last_launch_count() == 8  # 4 x (fold table + kernel)
    finally:
        B.lib().b2b_set_kernel_variant(0)
    assert rel(B.to_numpy(xs3), xo) <= RTOL and rel(B.to_numpy(ljf3), ljo) <= RTOL


def test_columnwise_sums_over_columns(B):
    """columnwise(f): logabsdetjac is the SUM over columns (src/interface.jl:71-78)."""
    rng = np.random.default_rng(21)
    D, N = 32, 3001
    lay, olay = make_case("radial", D, rng)
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)
    f = B.columnwise(lay)
    y, tot = B.with_logabsdet_jacobian(f, xd)
    yo, ljo = olay.forward(x.astype(np.float64))
    assert rel(B.to_numpy(y), yo) <= RTOL
    assert abs(float(tot) - ljo.sum()) <= 1e-5 * abs(ljo.sum())
    assert abs(float(B.logabsdetjac(f, xd)) - ljo.sum()) <= 1e-5 * abs(ljo.sum())
    xi, toti = B.with_logabsdet_jacobian(B.inverse(f), y)
    assert rel(B.to_numpy(xi), x) <= 1e-4 and abs(float(toti) + ljo.sum()) <= 1e-4 * abs(ljo.sum())


@pytest.mark.parametrize("D,N", [(32, 5000), (256, 4097), (10, 333)])
def test_batchnorm_training_mode(B, D, N):
    """InvertibleBatchNorm with istraining() == true (normalise.jl:51-60): batch statistics, moving-average update
    with the n/(n-1) correction, output and logjac from the batch statistics."""
    rng = np.random.default_rng(D)
    b, logs = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
    m0, v0 = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    x = (rng.standard_normal((D, N)) * rng.uniform(0.5, 2.0, D)[:, None] + rng.standard_normal(D)[:, None] * 3).astype(f32)
    bn = B.InvertibleBatchNorm(b=b, logs=logs, m=m0, v=v0, training=True)
    y, lj = B.with_logabsdet_jacobian(bn, B.from_numpy(x))
    obn = O.BatchNormParams(b.astype(np.float64), logs.astype(np.float64), m0.astype(np.float64), v0.astype(np.float64),
                            np.float64(f32(1e-5)), np.float64(f32(0.1)))
    yo, ljo, (m1, v1) = O.batchnorm_forward(obn, x.astype(np.float64), training=True)
    assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL
    assert rel(B.to_numpy(bn.m), m1) <= RTOL and rel(B.to_numpy(bn.v), v1) <= RTOL  # moving statistics updated in place
    # eval mode afterwards uses the UPDATED moving statistics
    bn.training = False
    y2, _ = B.with_logabsdet_jacobian(bn, B.from_numpy(x))
    ye, _ = O.batchnorm_forward(O.BatchNormParams(obn.b, obn.logs, m1, v1, obn.eps, obn.mtm), x.astype(np.float64))
    assert rel(B.to_numpy(y2), ye) <= RTOL
    with pytest.raises(RuntimeError, match="channels"):
        B.InvertibleBatchNorm(D + 1, training=True).train_forward(B.from_numpy(x))


@pytest.mark.parametrize("D", [128, 64, 10])
def test_edge_shapes_strides_alignment(B, D):
    """Empty / single-column / ragged batches, padded leading dimension, misaligned base pointers (these take the
    scalar-load build of the lane-group kernel), in-place evaluation, NaN columns staying local."""
    import torch

    rng = np.random.default_rng(D + 1)
    pairs = [make_case(k, D, rng) for k in ("planar", "radial", "batchnorm")]
    flow = B.Composed(*[p[0] for p in pairs])
    olayers = [p[1] for p in pairs]
    # N = 0: nothing is launched, empty outputs
    y0, lj0 = B.with_logabsdet_jacobian(flow, B.colmajor_empty(D, 0))
    assert y0.shape == (D, 0) and lj0.shape == (0,)
    for N in (1, 31, 33, 257):
        x = rng.standard_normal((D, N)).astype(f32)
        y, lj = B.with_logabsdet_jacobian(flow, B.from_numpy(x))
        yo, ljo = O.chain_forward(olayers, x.astype(np.float64))
        assert rel(B.to_numpy(y).reshape(D, N), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL, N
    N = 515
    x = rng.standard_normal((D, N)).astype(f32)
    yo, ljo = O.chain_forward(olayers, x.astype(np.float64))
    for pad in (4, 1):  # ld = D + 4 keeps 16-byte alignment; ld = D + 1 does not
        buf = torch.zeros((N, D + pad), device="cuda")
        xv = buf[:, :D].t()  # shape (D, N), strides (1, D + pad)
        xv.copy_(B.from_numpy(x))
        obuf = torch.full((N, D + pad), 7.0, device="cuda")
        yv = obuf[:, :D].t()
        y, lj = B.run_chain(flow, xv, y=yv)
        assert rel(B.to_numpy(yv), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL, pad
        assert bool((obuf[:, D:] == 7.0).all()), "padding between columns was overwritten"
    # misaligned base pointer (offset by one float)
    flat = torch.zeros(D * N + 1, device="cuda")
    xm = flat[1:].view(N, D).t()
    xm.copy_(B.from_numpy(x))
    y, lj = B.with_logabsdet_jacobian(flow, xm)
    assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL
    # in place (y aliases x)
    xi = B.from_numpy(x)
    y, lj = B.with_logabsdet_jacobian_(flow, xi)
    assert y.data_ptr() == xi.data_ptr() and rel(B.to_numpy(xi), yo) <= RTOL
    # a NaN column stays a NaN column and does not leak into its neighbours
    xn = x.copy()
    xn[:, 100] = np.nan
    y, lj = B.with_logabsdet_jacobian(flow, B.from_numpy(xn))
    yh, ljh = B.to_numpy(y), B.to_numpy(lj)
    assert np.isnan(yh[:, 100]).all() and np.isnan(ljh[100])
    keep = np.arange(N) != 100
    assert rel(yh[:, keep], yo[:, keep]) <= RTOL and rel(ljh[keep], ljo[keep]) <= RTOL


@pytest.mark.parametrize("N", [1, 63, 64, 65, 200])
def test_coupling_tc_ragged_batches(B, N):
    rng = np.random.default_rng(N)
    D = 256
    idx1, idx2 = list(range(1, 129)), list(range(129, 257))
    W = (rng.standard_normal((256, 128)) * 0.2 / np.sqrt(128)).astype(f32)
    c = (rng.standard_normal(256) * 0.1).astype(f32)
    cl = B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2))
    ol = O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c))
    x = rng.standard_normal((D, N)).astype(f32)
    y, lj = B.with_logabsdet_jacobian(cl, B.from_numpy(x))
    # whole tiles: W preparation + tensor-core kernel; the < 64 ragged columns: exact-fp32 kernel
    assert B.lib().b2b_last_launch_count() == (2 if N >= 64 else 0) + (1 if N % 64 else 0)
    yo, ljo = ol.forward(x.astype(np.float64))
    assert rel(B.to_numpy(y).reshape(D, N), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL


@pytest.mark.parametrize("D", [32, 64, 128, 256])
def test_tma_kernel_matches_lane_group_kernel_on_ragged_batches(B, D):
    """The TMA-staged kernel (several tiles per warp, input ring shallower than the warp count, tail tiles) against the
    direct-load kernel, repeated to catch hand-off races (regression test for the buffer re-arm flags)."""
    import torch

    rng = np.random.default_rng(D)
    lay = [make_case("radial", D, rng)[0], make_case("batchnorm", D, rng)[0], make_case("planar", D, rng)[0]]
    flow = B.Composed(*lay)
    for N in (3001, 5000, 100_000):
        x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
        B.lib().b2b_set_kernel_variant(1)
        try:
            y0, l0 = B.with_logabsdet_jacobian(flow, x)
            t0 = torch.zeros((), dtype=torch.float64, device="cuda")
            B.run_chain(flow, x, want_y=False, sum_out=t0)
        finally:
            B.lib().b2b_set_kernel_variant(0)
        for _ in range(10):
            y1, l1 = B.with_logabsdet_jacobian(flow, x)
            t1 = torch.zeros((), dtype=torch.float64, device="cuda")
            B.run_chain(flow, x, want_y=False, sum_out=t1)
            assert float((y1 - y0).norm() / y0.norm()) <= 2e-6
            assert float((l1 - l0).norm() / l0.norm()) <= 2e-6
            assert abs(float(t1 - t0)) <= 1e-7 * abs(float(t0))


def _full_size_props(B, flow, olayers, D, N, sample=2048, rt_tol=1e-4):
    """Size-independent properties at a BASELINE config's FULL size + an oracle check on a column sample."""
    import torch

    gen = torch.Generator(device="cuda").manual_seed(D + 3)
    x = torch.randn((N, D), device="cuda", generator=gen).t()
    y, lj = B.with_logabsdet_jacobian(flow, x)
    assert bool(torch.isfinite(y).all()) and bool(torch.isfinite(lj).all())
    cols = np.sort(np.random.default_rng(D).choice(N, sample, replace=False))
    ct = torch.as_tensor(cols, device="cuda")
    yo, ljo = O.chain_forward(olayers, x[:, ct].cpu().numpy().astype(np.float64))
    assert rel(y[:, ct].cpu().numpy(), yo) <= RTOL and rel(lj[ct].cpu().numpy(), ljo) <= RTOL
    xi, lji = B.with_logabsdet_jacobian(B.inverse(flow), y)
    # the INVERSE outputs against the oracle on the column sample (float64 and float32 reference on the device's y)
    ys = y[:, ct].cpu().numpy()
    xo, ljio = O.chain_inverse(olayers, ys.astype(np.float64))
    xo32, ljio32 = O.chain_inverse(olayers, ys)
    gx, gl = gate(xo32, xo), gate(ljio32, ljio)
    assert rel(xi[:, ct].cpu().numpy(), xo) <= gx, (rel(xi[:, ct].cpu().numpy(), xo), gx)
    assert rel(lji[ct].cpu().numpy(), ljio) <= gl, (rel(lji[ct].cpu().numpy(), ljio), gl)
    # whole batch: inverse∘forward ≈ id and ires == (x, −logjac) as well as the float64 reference manages from this y
    # (forward rounding amplified by the inverse's conditioning, measured on the sample), plus the inverse's own gate
    xs = x[:, ct].cpu().numpy()
    rt_x = 2 * (rel(xo, xs) + gx)
    rt_l = 2 * (rel(ljio, -ljo) + gl)
    assert rt_x <= rt_tol and rt_l <= rt_tol, (rt_x, rt_l)  # rt_tol documents how ill-conditioned the config may be
    assert float((xi - x).norm() / x.norm()) <= rt_x
    assert float((lji + lj).norm()) <= rt_l * max(float(lj.norm()), 1.0)
    td = B.transformed(B.MvNormal(D), flow)
    tot, lp = B.logpdf_sum(td, y)
    lpo = O.transformed_logpdf(olayers, np.zeros(D), np.ones(D), ys.astype(np.float64))
    lpo32 = O.transformed_logpdf(olayers, np.zeros(D, f32), np.ones(D, f32), ys)
    assert rel(lp[ct].cpu().numpy(), lpo) <= gate(lpo32, lpo), (rel(lp[ct].cpu().numpy(), lpo), rel(lpo32, lpo))
    # logpdf(td, y) = logpdf(base, x) − logjac(x)  (test/normalising_flows.jl:97-111), here for the whole batch
    base = -0.5 * (D * math.log(2 * math.pi)) - 0.5 * (x.double() ** 2).sum(0)
    ref = (base - lj.double())
    assert float((lp.double() - ref).norm() / ref.norm()) <= max(rt_x, rt_l)
    assert abs(float(tot) - float(lp.double().sum())) <= 1e-9 * abs(float(tot))
    return x, y, lj


def test_full_size_properties_config3_radial(B):
    """BASELINE config 3 at full size: 6 x RadialLayer, D = 64, N = 2^20, forward + inverse."""
    rng = np.random.default_rng(200)
    pairs = [make_case("radial", 64, np.random.default_rng(200 + l)) for l in range(6)]
    _full_size_props(B, B.Composed(*[p[0] for p in pairs]), [p[1] for p in pairs], 64, 1 << 20, rt_tol=2e-3)


def test_full_size_properties_config4_rqs(B):
    """BASELINE config 4 at full size: RationalQuadraticSpline K = 8, D = 32, N = 2^19 (about 5 % of the elements
    outside the box)."""
    import torch

    lay, olay = make_case("rqs", 32, np.random.default_rng(300))
    D, N = 32, 1 << 19
    gen = torch.Generator(device="cuda").manual_seed(4)
    x = (torch.randn((N, D), device="cuda", generator=gen) * 1.5).t()
    y, lj = B.with_logabsdet_jacobian(lay, x)
    outside = (x.abs() >= 3.0)
    assert 0.02 < float(outside.float().mean()) < 0.08
    assert bool((y[outside] == x[outside]).all())  # identity outside the box, bit for bit
    cols = np.sort(np.random.default_rng(1).choice(N, 4096, replace=False))
    ct = torch.as_tensor(cols, device="cuda")
    yo, ljo = olay.forward(x[:, ct].cpu().numpy().astype(np.float64))
    assert rel(y[:, ct].cpu().numpy(), yo) <= RTOL and rel(lj[ct].cpu().numpy(), ljo) <= RTOL
    xi, lji = B.with_logabsdet_jacobian(B.inverse(lay), y)
    assert float((xi - x).norm() / x.norm()) <= 1e-4 and float((lji + lj).norm() / lj.norm()) <= 1e-4
    # monotone: the spline preserves the order of any two inputs of the same row
    assert bool(((y[:, 1:] - y[:, :-1]) * (x[:, 1:] - x[:, :-1]) >= 0).all())


@pytest.mark.parametrize("D", [32, 64])
@pytest.mark.parametrize("K", [4, 8, 16, 32, 6, 2, 3, 10, 20, 31])
def test_rqs_bin_counts_and_raw_knots(B, D, K):
    """Specialised spline programs: table sizes for K in {4, 8, 16, 32} bins, any other K <= 32 in the next larger table
    (+inf probe padding), forward and inverse,
    against the float64 oracle -- with B-constructed knots and with RAW three-argument-constructor knots whose first
    knot is not -B, which reaches the k == 0 branches (rational_quadratic_spline.jl:331-343)."""
    rng = np.random.default_rng(7000 + 10 * K + D)
    N = 3001
    lay = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                    rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    W, H, Dv = lay.knots()
    cases = [(lay, W, H, Dv)]
    W2, H2 = W.copy(), H.copy()
    W2[:, 0] = -2.0 + 0.1 * rng.random(D).astype(f32)   # first knot right of -B = -3: points in (-3, W2[0]] hit k == 0
    H2[:, 0] = -2.2 + 0.1 * rng.random(D).astype(f32)
    W2[:, 1:] = np.maximum(W2[:, 1:], W2[:, :1] + 0.05 * np.arange(1, K + 1, dtype=f32))
    H2[:, 1:] = np.maximum(H2[:, 1:], H2[:, :1] + 0.05 * np.arange(1, K + 1, dtype=f32))
    W2[:, -1], H2[:, -1] = 3.0, 3.0
    W2, H2 = np.sort(W2, axis=1), np.sort(H2, axis=1)
    cases.append((B.RationalQuadraticSpline(W2, H2, Dv), W2, H2, Dv))
    for lay_, W_, H_, D_ in cases:
        olay = O.Layer("rqs", dict(widths=W_, heights=H_, derivs=D_))
        x = (rng.standard_normal((D, N)) * 1.6).astype(f32)
        x[:, 0] = W_[:, min(2, K)]          # a point exactly on a knot belongs to the bin on its left
        x[:, 1], x[:, 2] = W_[:, -1], -W_[:, -1]  # the box edges themselves are outside (x <= -B or x >= B, :322)
        xd = B.from_numpy(x)
        y, lj = B.with_logabsdet_jacobian(lay_, xd)
        yo, ljo = olay.forward(x.astype(np.float64))
        assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL, (K, D, rel(B.to_numpy(y), yo), rel(B.to_numpy(lj), ljo))
        out = np.abs(x) >= W_[:, -1:]
        assert np.array_equal(B.to_numpy(y)[out], x[out])
        # inverse: the exact box edges are left out (widths[end] and heights[end] may differ by an ulp, which puts
        # y = ±widths[end] into a zero-width k == 0 bin of the HEIGHT knots -- 0/0 in the reference as well)
        yh = B.to_numpy(y).copy()
        yh[:, 1], yh[:, 2] = 1.01 * H_[:, -1], -1.01 * H_[:, -1]
        xi, lji = B.with_logabsdet_jacobian(B.inverse(lay_), B.from_numpy(yh))
        xo, ljio = olay.inverse(yh.astype(np.float64))
        assert rel(B.to_numpy(xi), xo) <= RTOL and rel(B.to_numpy(lji), ljio) <= RTOL, (K, D, rel(B.to_numpy(xi), xo), rel(B.to_numpy(lji), ljio))
        assert np.array_equal(B.to_numpy(xi)[:, 1:3], yh[:, 1:3])


def test_full_size_properties_config5_realnvp_share(B):
    """BASELINE config 5, one GPU's share at 8-way sharding: 4 x (affine Coupling + InvertibleBatchNorm), D = 256,
    N = 2^19 columns."""
    rng = np.random.default_rng(400)
    D = 256
    dev_layers, ora_layers = [], []
    for l in range(4):
        first = l % 2 == 0
        idx1 = list(range(1, 129)) if first else list(range(129, 257))
        idx2 = list(range(129, 257)) if first else list(range(1, 129))
        W = (rng.standard_normal((256, 128)) * 0.05 / np.sqrt(128)).astype(f32)
        c = np.zeros(256, f32)
        dev_layers.append(B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2)))
        ora_layers.append(O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c)))
        b, logs, m = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
        v = rng.uniform(0.5, 1.5, D).astype(f32)
        dev_layers.append(B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v))
        ora_layers.append(O.Layer("batchnorm", dict(bn=O.BatchNormParams(b, logs, m, v, f32(1e-5), f32(0.1)))))
    _full_size_props(B, B.Composed(*dev_layers), ora_layers, D, 1 << 19, sample=1024)


@pytest.mark.parametrize("D", [128, 64, 32])
@pytest.mark.parametrize("L", [1, 3, 8, 11])
def test_planar_chain_with_host_resident_parameters(B, D, L):
    """PlanarLayers whose parameters stay in HOST memory (the reference's residency) on a device batch:
    b2b_planar_chain_hostparams_f32 -- same results as the device-parameter chain and the oracle."""
    import torch

    rng = np.random.default_rng(1000 * D + L)
    N = 2500 + L  # ragged: not a multiple of the 32-column tile
    pairs = [make_case("planar", D, rng) for _ in range(L)]
    dev_flow = B.Composed(*[p[0] for p in pairs])
    host_flow = B.Composed(*[p[0].to("cpu") for p in pairs])
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)
    y, lj = B.with_logabsdet_jacobian(host_flow, xd)
    assert B.lib().b2b_last_launch_count() == {1: 1, 3: 1, 8: 1, 11: 2}[L]
    yo, ljo = O.chain_forward([p[1] for p in pairs], x.astype(np.float64))
    assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL
    yd, ljd = B.with_logabsdet_jacobian(dev_flow, xd)
    assert rel(B.to_numpy(y), B.to_numpy(yd)) <= 2e-6 and rel(B.to_numpy(lj), B.to_numpy(ljd)) <= 2e-6
    # transform-only / logabsdetjac-only (the latter needs one launch: L <= 8)
    assert np.array_equal(B.to_numpy(B.transform(host_flow, xd)), B.to_numpy(y))
    if L <= 8:
        assert np.array_equal(B.to_numpy(B.logabsdetjac(host_flow, xd)), B.to_numpy(lj))
    # inverse chain (find_alpha per layer), in place + accumulating
    xi, lji = B.with_logabsdet_jacobian(B.inverse(host_flow), y)
    xid, ljid = B.with_logabsdet_jacobian(B.inverse(dev_flow), y)
    # both device paths (kernel-argument parameters + safeguarded iteration / shared-memory parameters + root table)
    # against the float64 oracle inverse of the SAME y, and against each other
    xo, ljio = O.chain_inverse([p[1] for p in pairs], B.to_numpy(y).astype(np.float64))
    for xx, ll in ((xi, lji), (xid, ljid)):
        assert rel(B.to_numpy(xx), xo) <= RTOL and rel(B.to_numpy(ll), ljio) <= RTOL, (rel(B.to_numpy(xx), xo), rel(B.to_numpy(ll), ljio))
    assert rel(B.to_numpy(xi), B.to_numpy(xid)) <= 5e-6 and rel(B.to_numpy(lji), B.to_numpy(ljid)) <= 5e-6
    assert rel(B.to_numpy(xi), x) <= 1e-4 and rel(B.to_numpy(lji), -ljo) <= 1e-4
    buf, acc = B.from_numpy(x), torch.full((N,), 0.5, dtype=torch.float32, device="cuda")
    buf, acc = B.with_logabsdet_jacobian_(host_flow, buf, None, acc)
    assert np.array_equal(B.to_numpy(buf), B.to_numpy(y))
    assert rel(B.to_numpy(acc), B.to_numpy(lj) + 0.5) <= 2e-6


def test_host_resident_parameters_unsupported_cases_fail_loudly(B):
    rng = np.random.default_rng(5)
    pl, _ = make_case("planar", 128, rng)
    rd, _ = make_case("radial", 128, rng)
    xd = B.from_numpy(rng.standard_normal((128, 64)).astype(f32))
    with pytest.raises(B.B2BError):  # mixed residency / non-planar layers
        B.with_logabsdet_jacobian(B.Composed(pl.to("cpu"), rd), xd)
    pl10, _ = make_case("planar", 10, rng)
    with pytest.raises(B.B2BError):  # D outside {32, 64, 128}: no silent fallback
        B.with_logabsdet_jacobian(pl10.to("cpu"), B.from_numpy(rng.standard_normal((10, 64)).astype(f32)))


@pytest.mark.parametrize("D", [128, 64, 32])
@pytest.mark.parametrize("L", [1, 3, 5, 6, 7, 8])
def test_constant_bank_planar_chain_matches_interpreter_and_oracle(B, D, L):
    """Segments of <= 8 PlanarLayers with device-resident parameters run as one unrolled program
    (b2b_planar_const.cu): same results as the layer interpreter and the oracle, mixed directions."""
    rng = np.random.default_rng(77 * D + L)
    N = 4000 + 3 * L
    pairs = [make_case("planar", D, rng) for _ in range(L)]
    # mix forward and inverse layers in one chain
    flow = B.Composed(*[B.inverse(p[0]) if i % 3 == 1 else p[0] for i, p in enumerate(pairs)])
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)
    lib = B.lib()
    try:
        assert lib.b2b_set_kernel_variant(3) == 0
        y3, lj3 = B.with_logabsdet_jacobian(flow, xd)
        assert lib.b2b_last_launch_count() == 1
        assert lib.b2b_set_kernel_variant(2) == 0
        y2, lj2 = B.with_logabsdet_jacobian(flow, xd)
        assert lib.b2b_last_launch_count() == 1
    finally:
        lib.b2b_set_kernel_variant(0)
    y0, lj0 = B.with_logabsdet_jacobian(flow, xd)  # auto picks the unrolled planar kernel
    assert np.array_equal(B.to_numpy(y0), B.to_numpy(y3)) and np.array_equal(B.to_numpy(lj0), B.to_numpy(lj3))
    assert rel(B.to_numpy(y3), B.to_numpy(y2)) <= 5e-6 and rel(B.to_numpy(lj3), B.to_numpy(lj2)) <= 5e-6  # two kernels, each gated against the oracle below
    # oracle: forward layers forward, inverse layers through the oracle inverse -- in float64, and in float32 for the gate
    def mixed(x0):
        z, ljo = x0, np.zeros(N, x0.dtype)
        for i, p in enumerate(pairs):
            z, l1 = (O.chain_inverse if i % 3 == 1 else O.chain_forward)([p[1]], z)
            ljo = ljo + l1
        return z, ljo

    z, ljo = mixed(x.astype(np.float64))
    z32, ljo32 = mixed(x)
    assert rel(B.to_numpy(y3), z) <= gate(z32, z) and rel(B.to_numpy(lj3), ljo) <= gate(ljo32, ljo), (
        rel(B.to_numpy(y3), z), rel(z32, z), rel(B.to_numpy(lj3), ljo), rel(ljo32, ljo))
    fwd = B.Composed(*[p[0] for p in pairs])
    olayers = [p[1] for p in pairs]
    yf, ljf = B.with_logabsdet_jacobian(fwd, xd)
    yo, lo = O.chain_forward(olayers, x.astype(np.float64))
    assert rel(B.to_numpy(yf), yo) <= RTOL and rel(B.to_numpy(ljf), lo) <= RTOL
    # all-inverse program of exactly L layers, and the logpdf program (terminal MvNormal) of the same length
    yh = B.to_numpy(yf)
    xi, lji = B.with_logabsdet_jacobian(B.inverse(fwd), yf)
    assert lib.b2b_last_launch_count() == 1
    xo, ljio = O.chain_inverse(olayers, yh.astype(np.float64))
    xo32, ljio32 = O.chain_inverse(olayers, yh)
    assert rel(B.to_numpy(xi), xo) <= gate(xo32, xo) and rel(B.to_numpy(lji), ljio) <= gate(ljio32, ljio)
    mu, sigma = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 2.0, D).astype(f32)
    lp = B.to_numpy(B.logpdf(B.transformed(B.MvNormal(D, mu, sigma), fwd), yf))
    assert lib.b2b_last_launch_count() == 1
    lpo = O.transformed_logpdf(olayers, mu.astype(np.float64), sigma.astype(np.float64), yh.astype(np.float64))
    assert rel(lp, lpo) <= gate(O.transformed_logpdf(olayers, mu, sigma, yh), lpo)


def test_constant_bank_slot_is_safe_across_streams(B):
    """The __constant__ parameter slot is per-device state: launches from different streams with different flows
    are ordered by the library (event), results never mix."""
    import torch

    rng = np.random.default_rng(99)
    D, N = 128, 1 << 16
    flows, outs, refs = [], [], []
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    for k in range(4):
        pairs = [make_case("planar", D, rng) for _ in range(8)]
        flows.append(B.Composed(*[p[0] for p in pairs]))
    lib = B.lib()
    lib.b2b_set_kernel_variant(2)
    try:
        for f in flows:
            refs.append(tuple(B.to_numpy(t) for t in B.with_logabsdet_jacobian(f, x)))
    finally:
        lib.b2b_set_kernel_variant(0)
    streams = [torch.cuda.Stream() for _ in flows]
    torch.cuda.synchronize()
    for rep in range(5):
        outs = []
        for f, s in zip(flows, streams):
            with torch.cuda.stream(s):
                outs.append(B.with_logabsdet_jacobian(f, x))
        torch.cuda.synchronize()
        for (y, lj), (yr, ljr) in zip(outs, refs):
            assert rel(B.to_numpy(y), yr) <= 2e-6 and rel(B.to_numpy(lj), ljr) <= 2e-6


@pytest.mark.parametrize("D,L", [(128, 8), (64, 5), (32, 2)])
def test_constant_bank_logpdf_of_planar_flow(B, D, L):
    """logpdf(transformed(MvNormal, planar flow), y) (transformed_distribution.jl:165-169): the all-inverse planar
    chain + base log-density (+ batch sum) through the constant-bank kernel = interpreter = oracle."""
    rng = np.random.default_rng(31 * D + L)
    N = 3000 + L
    pairs = [make_case("planar", D, rng) for _ in range(L)]
    flow = B.Composed(*[p[0] for p in pairs])
    mu, sigma = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 2.0, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu, sigma), flow)
    x = rng.standard_normal((D, N)).astype(f32)
    yo, ljo = O.chain_forward([p[1] for p in pairs], x.astype(np.float64))
    y = B.from_numpy(yo.astype(f32))
    lib = B.lib()
    res = {}
    try:
        for variant in (3, 2):
            assert lib.b2b_set_kernel_variant(variant) == 0
            lp = B.logpdf(td, y)
            n_launch = lib.b2b_last_launch_count()
            tot, lp2 = B.logpdf_sum(td, y)
            res[variant] = (B.to_numpy(lp), float(tot), B.to_numpy(lp2), n_launch)
    finally:
        lib.b2b_set_kernel_variant(0)
    assert res[3][3] == 1 and res[2][3] == 1
    assert rel(res[3][0], res[2][0]) <= 2e-6
    assert np.array_equal(res[3][0], res[3][2])
    assert abs(res[3][1] - float(res[3][0].astype(np.float64).sum())) <= 1e-9 * abs(res[3][1]) + 1e-6
    # oracle logpdf of the very batch the device saw (the float32-rounded y), in float64 and -- for the gate -- float32
    olayers, yh = [p[1] for p in pairs], B.to_numpy(y)
    lpo = O.transformed_logpdf(olayers, mu.astype(np.float64), sigma.astype(np.float64), yh.astype(np.float64))
    lpo32 = O.transformed_logpdf(olayers, mu, sigma, yh)
    assert rel(res[3][0], lpo) <= gate(lpo32, lpo) and rel(res[2][0], lpo) <= gate(lpo32, lpo), (rel(res[3][0], lpo), rel(lpo32, lpo))
    assert np.array_equal(B.to_numpy(B.logpdf(td, y)), res[3][0])  # auto = constant-bank path


@pytest.mark.parametrize("D", [128, 64, 32])
@pytest.mark.parametrize("L", [1, 3, 8])
def test_planar_chain_vjp_matches_oracle(B, D, L):
    """b2b_planar_chain_vjp_f32 (reverse mode of with_logabsdet_jacobian through a planar chain) against the
    float64 oracle VJP, which is itself pinned by finite differences of the forward oracle (CPU suite)."""
    import torch

    rng = np.random.default_rng(500 * D + L)
    N = 6000 + 7 * L  # ragged
    pairs = [make_case("planar", D, rng) for _ in range(L)]
    flow = B.Composed(*[p[0] for p in pairs])
    params = [(p[1].params["w"], p[1].params["u"], p[1].params["b"]) for p in pairs]
    x = rng.standard_normal((D, N)).astype(f32)
    ybar = rng.standard_normal((D, N)).astype(f32)
    ljbar = rng.standard_normal(N).astype(f32)
    xb_o, grads_o = O.planar_chain_vjp([(w.astype(np.float64), u.astype(np.float64), b.astype(np.float64)) for w, u, b in params],
                                       x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64))
    xd, ybd, ljd = B.from_numpy(x), B.from_numpy(ybar), torch.from_numpy(ljbar).cuda()
    xbar, grads = B.planar_chain_vjp(flow, xd, ybd, ljd)
    assert B.lib().b2b_last_launch_count() == 7
    assert rel(B.to_numpy(xbar), xb_o) <= RTOL
    for l in range(L):
        # parameter cotangents are sums of N float32 products: 2e-5 norm-wise
        assert rel(grads[l]["w"].cpu().numpy(), grads_o[l][0]) <= 2e-5, (l, "w")
        assert rel(grads[l]["u"].cpu().numpy(), grads_o[l][1]) <= 2e-5, (l, "u")
        assert abs(float(grads[l]["b"]) - float(grads_o[l][2])) <= 2e-5 * max(abs(float(grads_o[l][2])), np.sqrt(N))
    # inputs untouched; xbar-only call (no parameter cotangents), ljbar = None
    assert np.array_equal(B.to_numpy(xd), x) and np.array_equal(B.to_numpy(ybd), ybar)
    xbar2, g2 = B.planar_chain_vjp(flow, xd, ybd, None, want_param_grads=False)
    assert g2 is None and B.lib().b2b_last_launch_count() == 1
    xb_o2, _ = O.planar_chain_vjp([(w.astype(np.float64), u.astype(np.float64), b.astype(np.float64)) for w, u, b in params],
                                  x.astype(np.float64), ybar.astype(np.float64), np.zeros(N))
    assert rel(B.to_numpy(xbar2), xb_o2) <= RTOL
    # determinism of the reductions
    xbar3, grads3 = B.planar_chain_vjp(flow, xd, ybd, ljd)
    assert all(torch.equal(grads3[l][k], grads[l][k]) for l in range(L) for k in ("w", "u", "b"))


@pytest.mark.parametrize("D,L", [(128, 8), (64, 3), (32, 1)])
def test_planar_inverse_chain_vjp_matches_oracle(B, D, L):
    """Reverse mode of with_logabsdet_jacobian(inverse(flow), y) -- the logpdf / NLL training path
    (docs/src/flows.md:66-100), find_alpha differentiated with the reference's implicit rule -- vs the float64 oracle."""
    import torch

    rng = np.random.default_rng(900 * D + L)
    N = 5000 + L
    pairs = [make_case("planar", D, rng) for _ in range(L)]
    flow = B.Composed(*[p[0] for p in pairs])
    params = [tuple(p[1].params[k].astype(np.float64) for k in ("w", "u", "b")) for p in pairs]
    y = rng.standard_normal((D, N)).astype(f32)
    xbar = rng.standard_normal((D, N)).astype(f32)
    ljbar = rng.standard_normal(N).astype(f32)
    yb_o, grads_o = O.planar_inverse_chain_vjp(params, y.astype(np.float64), xbar.astype(np.float64), ljbar.astype(np.float64))
    ybar, grads = B.planar_chain_vjp(B.inverse(flow), B.from_numpy(y), B.from_numpy(xbar), torch.from_numpy(ljbar).cuda())
    assert rel(B.to_numpy(ybar), yb_o) <= 2e-5
    grads = grads[::-1]  # application order of inverse(flow) -> the flow's layer order
    for l in range(L):
        assert rel(grads[l]["w"].cpu().numpy(), grads_o[l][0]) <= 5e-5, (l, "w")
        assert rel(grads[l]["u"].cpu().numpy(), grads_o[l][1]) <= 5e-5, (l, "u")
        assert abs(float(grads[l]["b"]) - float(grads_o[l][2])) <= 5e-5 * max(abs(float(grads_o[l][2])), np.sqrt(N))


@pytest.mark.parametrize("D,flags", [(64, [0, 1, 1, 0]), (32, [0] * 9 + [1, 1, 0]), (128, [1, 0, 0, 1, 1])])
def test_planar_chain_vjp_mixed_directions_and_long_chains(B, D, flags):
    """PlanarLayers and Inverse(PlanarLayer)s in one chain, and chains of more than 8 layers: cut into runs of one
    direction (<= 8 layers) on the host side, each run differentiated by b2b_planar_chain_vjp_f32 -- against the float64
    oracle composed the same way."""
    import torch

    rng = np.random.default_rng(77 + D)
    N = 3000 + 11
    pairs = [make_case("planar", D, rng) for _ in flags]
    flow = B.Composed(*[B.inverse(p[0]) if f else p[0] for p, f in zip(pairs, flags)])
    P64 = [tuple(p[1].params[k].astype(np.float64) for k in ("w", "u", "b")) for p in pairs]
    x = rng.standard_normal((D, N)).astype(f32)
    ybar, ljbar = rng.standard_normal((D, N)).astype(f32), rng.standard_normal(N).astype(f32)
    # oracle: maximal runs of one direction, forward sweep for the run inputs, then the run VJPs last to first
    runs, i = [], 0
    while i < len(flags):
        j = i
        while j < len(flags) and flags[j] == flags[i]:
            j += 1
        runs.append((flags[i], list(range(i, j))))
        i = j
    ins, z = [], x.astype(np.float64)
    for f, idx in runs:
        ins.append(z)
        z = O.chain_inverse([pairs[k][1] for k in idx[::-1]], z)[0] if f else O.chain_forward([pairs[k][1] for k in idx], z)[0]
    cot, g_o = ybar.astype(np.float64), [None] * len(flags)
    for (f, idx), zin in zip(reversed(runs), reversed(ins)):
        if f:  # application order inv(A), inv(B) = inverse(Composed(B, A)): the oracle takes the flow's order
            cot, gr = O.planar_inverse_chain_vjp([P64[k] for k in idx[::-1]], zin, cot, ljbar.astype(np.float64))
            for k, g in zip(idx[::-1], gr):
                g_o[k] = g
        else:
            cot, gr = O.planar_chain_vjp([P64[k] for k in idx], zin, cot, ljbar.astype(np.float64))
            for k, g in zip(idx, gr):
                g_o[k] = g
    xbar, grads = B.planar_chain_vjp(flow, B.from_numpy(x), B.from_numpy(ybar), torch.from_numpy(ljbar).cuda())
    assert len(grads) == len(flags)
    assert rel(B.to_numpy(xbar), cot) <= 2e-5, rel(B.to_numpy(xbar), cot)
    for l in range(len(flags)):
        assert rel(grads[l]["w"].cpu().numpy(), g_o[l][0]) <= 5e-5, (l, "w")
        assert rel(grads[l]["u"].cpu().numpy(), g_o[l][1]) <= 5e-5, (l, "u")
        assert abs(float(grads[l]["b"]) - float(g_o[l][2])) <= 5e-5 * max(abs(float(g_o[l][2])), np.sqrt(N))


def test_planar_flow_trains_through_autograd(B):
    """The reference's training example (docs/src/flows.md:66-100: gradient descent on −Σ logpdf(transformed(base, flow),
    data)) with torch.autograd driving b2b_planar_chain_vjp_f32: gradients match the oracle, the loss goes down."""
    import torch

    torch.manual_seed(0)
    D, N, L = 32, 4096, 2
    gen = torch.Generator().manual_seed(3)
    flow = B.autograd.PlanarFlow(D, L, generator=gen, scale=1.0 / np.sqrt(D))
    data = B.from_numpy((np.random.default_rng(4).standard_normal((D, N)) * 1.5 + 0.3).astype(f32))

    def nll():
        x, lj = flow.inverse(data)  # logpdf(td, y) = logpdf(base, x) + logjac of the inverse chain
        base = -0.5 * (x * x).sum(dim=0) - 0.5 * D * math.log(2 * math.pi)  # MvNormal(zeros, I), example-level glue
        return -(base + lj).mean()

    loss0 = nll()
    loss0.backward()
    # oracle gradient of the same objective
    params = [(w.detach().cpu().numpy().astype(np.float64), u.detach().cpu().numpy().astype(np.float64),
               b.detach().cpu().numpy().astype(np.float64)) for w, u, b in zip(flow.w, flow.u, flow.b)]
    y64 = B.to_numpy(data).astype(np.float64)
    z, lj = y64, np.zeros(N)
    for (w, u, b) in reversed(params):
        z, l1 = O.planar_inverse(w, u, b, z)
        lj = lj + l1
    xbar = z / N          # d(−mean(base))/dx = x/N
    ljbar = -np.ones(N) / N
    _, grads_o = O.planar_inverse_chain_vjp(params, y64, xbar, ljbar)
    for l in range(L):
        assert rel(flow.w[l].grad.cpu().numpy(), grads_o[l][0]) <= 1e-4
        assert rel(flow.u[l].grad.cpu().numpy(), grads_o[l][1]) <= 1e-4
        assert abs(float(flow.b[l].grad) - float(grads_o[l][2])) <= 1e-4 * max(1.0, abs(float(grads_o[l][2])))
    opt = torch.optim.SGD(flow.parameters(), lr=5e-2)
    for _ in range(30):
        opt.zero_grad()
        loss = nll()
        loss.backward()
        opt.step()
    assert float(nll()) < float(loss0) - 1e-3
    # forward direction is differentiable too (sampling path): d/dx of Σ y + Σ logjac
    x = B.from_numpy(np.random.default_rng(5).standard_normal((D, 256)).astype(f32)).requires_grad_(True)
    yy, ll = flow(x)
    (yy.sum() + ll.sum()).backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()


def test_autograd_small_dimension_flow_like_the_reference_example(B):
    """docs/src/flows.md:40-110 uses PlanarLayer(2) on 1000 points: D = 2 runs embedded in the D = 32 reverse-mode
    kernels (zero-padded rows leave a planar layer unchanged); gradients equal the oracle's."""
    import torch

    rng = np.random.default_rng(8)
    D, N, L = 2, 1000, 2
    flow = B.autograd.PlanarFlow(D, L, generator=torch.Generator().manual_seed(1))
    data = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    x, lj = flow.inverse(data)
    loss = -((-0.5 * (x * x).sum(dim=0) - 0.5 * D * math.log(2 * math.pi)) + lj).sum()
    loss.backward()
    params = [(w.detach().cpu().numpy().astype(np.float64), u.detach().cpu().numpy().astype(np.float64),
               b.detach().cpu().numpy().astype(np.float64)) for w, u, b in zip(flow.w, flow.u, flow.b)]
    y64 = B.to_numpy(data).astype(np.float64)
    z = y64
    for (w, u, b) in reversed(params):
        z, _ = O.planar_inverse(w, u, b, z)
    _, grads_o = O.planar_inverse_chain_vjp(params, y64, z, -np.ones(N))
    for l in range(L):
        assert rel(flow.w[l].grad.cpu().numpy(), grads_o[l][0]) <= 1e-4
        assert rel(flow.u[l].grad.cpu().numpy(), grads_o[l][1]) <= 1e-4
        assert abs(float(flow.b[l].grad) - float(grads_o[l][2])) <= 1e-4 * max(1.0, abs(float(grads_o[l][2])))



@pytest.mark.parametrize("D,L", [(64, 6), (32, 1), (128, 8), (10, 3), (50, 5), (100, 2)])
def test_radial_chain_vjp_matches_oracle(B, D, L):
    """b2b_radial_chain_vjp_f32 (reverse mode through radial_layer.jl:43-72) vs the float64 oracle VJP, itself pinned
    by finite differences of the forward oracle (CPU suite).  Cotangents are w.r.t. the RAW parameters α_, β, z_0."""
    import torch

    rng = np.random.default_rng(700 * D + L)
    N = 4001 + L
    pairs = [make_case("radial", D, rng) for _ in range(L)]
    flow = B.Composed(*[p[0] for p in pairs])
    params = [(p[1].params["alpha_raw"].astype(np.float64), p[1].params["beta"].astype(np.float64),
               p[1].params["z0"].astype(np.float64)) for p in pairs]
    x = rng.standard_normal((D, N)).astype(f32)
    ybar = rng.standard_normal((D, N)).astype(f32)
    ljbar = rng.standard_normal(N).astype(f32)
    xb_o, g_o = O.radial_chain_vjp(params, x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64))
    xbar, grads = B.radial_chain_vjp(flow, B.from_numpy(x), B.from_numpy(ybar), torch.from_numpy(ljbar).cuda())
    assert B.lib().b2b_last_launch_count() == 2
    assert rel(B.to_numpy(xbar), xb_o) <= 2e-5
    for l in range(L):
        scale = np.sqrt(N)
        assert abs(float(grads[l]["α_"]) - float(g_o[l][0])) <= 5e-5 * max(abs(float(g_o[l][0])), scale), (l, "alpha")
        assert abs(float(grads[l]["β"]) - float(g_o[l][1])) <= 5e-5 * max(abs(float(g_o[l][1])), scale), (l, "beta")
        assert rel(grads[l]["z_0"].cpu().numpy(), g_o[l][2]) <= 5e-5, (l, "z0")
    # determinism + ljbar = None
    xbar2, grads2 = B.radial_chain_vjp(flow, B.from_numpy(x), B.from_numpy(ybar), torch.from_numpy(ljbar).cuda())
    assert torch.equal(xbar2, xbar) and all(torch.equal(grads2[l][k], grads[l][k]) for l in range(L) for k in ("α_", "β", "z_0"))
    xb0, _ = B.radial_chain_vjp(flow, B.from_numpy(x), B.from_numpy(ybar), None)
    xb_o0, _ = O.radial_chain_vjp(params, x.astype(np.float64), ybar.astype(np.float64), np.zeros(N))
    assert rel(B.to_numpy(xb0), xb_o0) <= 2e-5


def test_radial_flow_autograd(B):
    """torch.autograd over b2b_radial_chain_vjp_f32: gradients of a scalar loss equal the oracle's."""
    import torch

    D, N, L = 10, 777, 2
    flow = B.autograd.RadialFlow(D, L, generator=torch.Generator().manual_seed(2))
    x = B.from_numpy(np.random.default_rng(9).standard_normal((D, N)).astype(f32)).requires_grad_(True)
    y, lj = flow(x)
    ((y * y).sum() * 0.5 + lj.sum()).backward()
    params = [(a.detach().cpu().numpy().astype(np.float64), b.detach().cpu().numpy().astype(np.float64),
               z.detach().cpu().numpy().astype(np.float64)) for a, b, z in zip(flow.alpha_, flow.beta, flow.z_0)]
    x64 = B.to_numpy(x.detach()).astype(np.float64)
    z = x64
    for (a, b, z0) in params:
        z, _ = O.radial_forward(a, b, z0, z)
    xb_o, g_o = O.radial_chain_vjp(params, x64, z, np.ones(N))
    assert rel(B.to_numpy(x.grad), xb_o) <= 5e-5
    for l in range(L):
        assert abs(float(flow.alpha_[l].grad) - float(g_o[l][0])) <= 1e-4 * max(1.0, abs(float(g_o[l][0])))
        assert abs(float(flow.beta[l].grad) - float(g_o[l][1])) <= 1e-4 * max(1.0, abs(float(g_o[l][1])))
        assert rel(flow.z_0[l].grad.cpu().numpy(), g_o[l][2]) <= 1e-4


def test_full_size_vjp_round_trip_property(B):
    """Size-independent property at BASELINE config-2 size (8 layers, D = 128, N = 2^20): pulling a cotangent back
    through inverse(flow) at y and then through flow at x returns it (J(inverse(f))(y) = J(f)(x)⁻¹), and the parameter
    cotangents are deterministic."""
    import torch

    rng = np.random.default_rng(123)
    D, N, L = 128, 1 << 20, 8
    pairs = [make_case("planar", D, rng) for _ in range(L)]
    flow = B.Composed(*[p[0] for p in pairs])
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((N, D), device="cuda", generator=gen).t()
    v = torch.randn((N, D), device="cuda", generator=gen).t()
    y, _ = B.with_logabsdet_jacobian(flow, x)
    u_, _ = B.planar_chain_vjp(B.inverse(flow), y, v, None, want_param_grads=False)
    back, grads = B.planar_chain_vjp(flow, x, u_, None)
    err = float((back - v).norm() / v.norm())
    assert err <= 2e-5, err
    _, grads2 = B.planar_chain_vjp(flow, x, u_, None)
    assert all(torch.equal(grads[l][k], grads2[l][k]) for l in range(L) for k in ("w", "u", "b"))
    assert all(torch.isfinite(grads[l][k]).all() for l in range(L) for k in ("w", "u", "b"))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,n1,idx", [(256, 128, "halves"), (256, 128, "swapped"), (64, 20, "scattered"), (10, 4, "scattered"),
                                      (64, 24, "scattered4"), (128, 32, "scattered4")])
def test_coupling_and_batchnorm_vjp_match_oracle(B, D, n1, idx, inv):
    """Reverse mode of the RealNVP layer kinds: b2b_coupling_affine_vjp_f32 (incl. the combine pullback: pass-through rows
    and arbitrary index lists) and b2b_batchnorm_eval_vjp_f32, both directions, against the finite-difference-pinned
    float64 oracle; deterministic; ragged N."""
    rng = np.random.default_rng(900 + D + n1 + int(inv))
    N = 1000 + 37
    if idx == "halves":
        idx1, idx2 = list(range(1, n1 + 1)), list(range(n1 + 1, D + 1))
    elif idx == "swapped":
        idx1, idx2 = list(range(D - n1 + 1, D + 1)), list(range(1, D - n1 + 1))
    else:
        perm = rng.permutation(D) + 1
        # two (four) pass-through rows, x2 rows unsorted; "scattered4": n1, n2 multiples of 4 = the float4 program with index lists
        idx1, idx2 = sorted(perm[:n1].tolist()), perm[n1:D - (4 if idx == "scattered4" else 2)].tolist()
    n2 = len(idx2)
    W = (rng.standard_normal((2 * n1, n2)) * 0.3 / np.sqrt(n2)).astype(f32)
    c = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    cl = B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2))
    x, ybar, ljbar = (rng.standard_normal((D, N)).astype(f32), rng.standard_normal((D, N)).astype(f32), rng.standard_normal(N).astype(f32))
    t = B.inverse(cl) if inv else cl
    import torch

    xbar, g = B.coupling_vjp(t, B.from_numpy(x), B.from_numpy(ybar), torch.as_tensor(ljbar, device="cuda"))
    xo, Wo, co = O.coupling_affine_vjp(idx1, idx2, W.astype(np.float64), c.astype(np.float64), x.astype(np.float64),
                                       ybar.astype(np.float64), ljbar.astype(np.float64), inverse=inv)
    assert rel(B.to_numpy(xbar), xo) <= RTOL, rel(B.to_numpy(xbar), xo)
    assert rel(B.to_numpy(g["W"]), Wo) <= RTOL and rel(B.to_numpy(g["c"]), co) <= RTOL, (rel(B.to_numpy(g["W"]), Wo), rel(B.to_numpy(g["c"]), co))
    xbar2, g2 = B.coupling_vjp(t, B.from_numpy(x), B.from_numpy(ybar), torch.as_tensor(ljbar, device="cuda"))
    assert torch.equal(xbar, xbar2) and torch.equal(g["W"], g2["W"]) and torch.equal(g["c"], g2["c"])  # deterministic
    # eval-mode BatchNorm
    b, logs, m = (rng.standard_normal(D) * 0.3).astype(f32), (rng.standard_normal(D) * 0.3).astype(f32), (rng.standard_normal(D) * 0.3).astype(f32)
    v = rng.uniform(0.5, 1.5, D).astype(f32)
    bn = B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v)
    tb = B.inverse(bn) if inv else bn
    xb, gb = B.batchnorm_vjp(tb, B.from_numpy(x), B.from_numpy(ybar), torch.as_tensor(ljbar, device="cuda"))
    obn = O.BatchNormParams(b.astype(np.float64), logs.astype(np.float64), m.astype(np.float64), v.astype(np.float64), np.float64(np.float32(1e-5)), np.float64(0.1))
    xbo, bo, lo = O.batchnorm_eval_vjp(obn, x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64), inverse=inv)
    assert rel(B.to_numpy(xb), xbo) <= RTOL and rel(B.to_numpy(gb["b"]), bo) <= RTOL and rel(B.to_numpy(gb["logs"]), lo) <= RTOL, (
        rel(B.to_numpy(xb), xbo), rel(B.to_numpy(gb["b"]), bo), rel(B.to_numpy(gb["logs"]), lo))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,K", [(32, 8), (64, 8), (10, 8), (64, 32), (200, 4), (256, 63), (64, 11)])
def test_rqs_vjp_matches_oracle(B, D, K, inv):
    """Reverse mode of the RationalQuadraticSpline (b2b_rqs_vjp_f32), both directions, against the finite-difference-pinned
    float64 oracle: input cotangent and the cotangents of the processed widths / heights / derivatives; raw-knot splines
    reach the k == 0 scatter rule (x_k = −widths[end]); deterministic; ragged N; elements outside the box pass ȳ through."""
    import torch

    rng = np.random.default_rng(1200 + D + K + int(inv))
    N = 4000 + 13
    lay = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                    rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    W, H, Dv = lay.knots()
    W2, H2 = W.copy(), H.copy()
    W2[:, 0], H2[:, 0] = -2.5, -2.6  # first knot right of −B: points in (−3, W2[0]] are in the k == 0 bin
    W2, H2 = np.sort(np.maximum(W2, W2[:, :1]), axis=1), np.sort(np.maximum(H2, H2[:, :1]), axis=1)
    W2 += 1e-3 * np.arange(K + 1, dtype=f32)
    H2 += 1e-3 * np.arange(K + 1, dtype=f32)
    for lay_, W_, H_ in ((lay, W, H), (B.RationalQuadraticSpline(W2, H2, Dv), W2, H2)):
        x = (rng.standard_normal((D, N)) * 1.7).astype(f32)
        ybar, ljbar = rng.standard_normal((D, N)).astype(f32), rng.standard_normal(N).astype(f32)
        t = B.inverse(lay_) if inv else lay_
        a = (x * (H_[:, -1:] / W_[:, -1:])).astype(f32) if inv else x  # observed batch for the inverse direction
        ad, yd, ld = B.from_numpy(a), B.from_numpy(ybar), torch.as_tensor(ljbar, device="cuda")
        xbar, g = B.rqs_vjp(t, ad, yd, ld)
        args64 = [v.astype(np.float64) for v in (W_, H_, Dv, a, ybar, ljbar)]
        ref = O.rqs_vjp(*args64, inverse=inv)
        own = O.rqs_vjp(W_, H_, Dv, a, ybar, ljbar, inverse=inv)  # the float32 oracle's own error sets the gate
        got = (B.to_numpy(xbar), B.to_numpy(g["widths"]), B.to_numpy(g["heights"]), B.to_numpy(g["derivatives"]))
        for name, gv, rv, ov in zip(("xbar", "widths", "heights", "derivatives"), got, ref, own):
            assert gv.shape == rv.shape and np.isfinite(gv).all(), name
            assert rel(gv, rv) <= gate(ov, rv), (name, D, K, inv, rel(gv, rv), rel(ov, rv))
        S = H_ if inv else W_
        out = np.abs(a) >= S[:, -1:]
        assert out.any() and np.array_equal(got[0][out], ybar[out])
        xbar2, g2 = B.rqs_vjp(t, ad, yd, ld)
        assert torch.equal(xbar, xbar2) and all(torch.equal(g[k_], g2[k_]) for k_ in g)  # deterministic
        xbar3, g3 = B.rqs_vjp(t, ad, yd, None)                                            # ljbar = NULL means zeros
        r0 = O.rqs_vjp(*args64[:5], None, inverse=inv)
        assert rel(B.to_numpy(xbar3), r0[0]) <= 1e-4 and rel(B.to_numpy(g3["derivatives"]), r0[3]) <= 1e-4


@pytest.mark.parametrize("inv", [False, True])
def test_spline_layer_trains_through_autograd(B, inv):
    """autograd.SplineLayer: gradients of a scalar objective w.r.t. the RAW spline parameters (through the constructor's
    softmax / cumsum / softplus in torch and b2b_rqs_vjp_f32 on the device) equal the float64 oracle's -- oracle VJP of the
    spline chained with a float64 torch restatement of the constructor -- and a few SGD steps lower the objective."""
    import torch

    torch.manual_seed(5)
    D, K, N = 32, 8, 4096
    lay = B.autograd.SplineLayer(D, K, 3.0)
    x = (torch.randn((N, D), device="cuda") * 1.4).t()
    x.requires_grad_(True)
    cy, cl = torch.randn((N, D), device="cuda").t(), torch.randn(N, device="cuda")

    def objective():
        y, lj = (lay.inverse if inv else lay.forward)(x)
        return (y * cy).sum() + (lj * cl).sum()

    loss = objective()
    loss.backward()
    # float64 reference: oracle VJP for the knots, torch float64 autograd for the constructor
    w64, h64, d64 = [p.detach().double().cpu().requires_grad_(True) for p in (lay.w, lay.h, lay.d)]
    zero, one = torch.zeros((D, 1), dtype=torch.float64), torch.ones((D, 1), dtype=torch.float64)
    W64 = 6.0 * torch.cumsum(torch.cat([zero, torch.softmax(w64, 1)], 1), 1) - 3.0
    H64 = 6.0 * torch.cumsum(torch.cat([zero, torch.softmax(h64, 1)], 1), 1) - 3.0
    D64 = torch.cat([one, torch.nn.functional.softplus(d64), one], 1)
    # the spline is evaluated at the knots the device used (the float32 constructor's): next to a knot the cotangents
    # move by 1e-4 when the knot moves by one float32 ulp, which is not the kernel's error
    Wd, Hd, Dd = [k.detach().cpu().numpy().astype(np.float64) for k in lay.knots()]
    assert rel(Wd, W64.detach().numpy()) <= 1e-6 and rel(Dd, D64.detach().numpy()) <= 1e-6
    xb_o, Wb, Hb, Db = O.rqs_vjp(Wd, Hd, Dd, x.detach().cpu().numpy().astype(np.float64), cy.cpu().numpy().astype(np.float64),
                                 cl.cpu().numpy().astype(np.float64), inverse=inv)
    torch.autograd.backward([W64, H64, D64], [torch.from_numpy(Wb), torch.from_numpy(Hb), torch.from_numpy(Db)])
    assert rel(x.grad.cpu().numpy(), xb_o) <= 2e-5, rel(x.grad.cpu().numpy(), xb_o)
    for par, ref in ((lay.w, w64), (lay.h, h64), (lay.d, d64)):
        assert rel(par.grad.cpu().numpy(), ref.grad.numpy()) <= 5e-5, rel(par.grad.cpu().numpy(), ref.grad.numpy())
    opt = torch.optim.SGD(lay.parameters(), lr=1e-4)
    l0 = float(loss)
    for _ in range(5):
        opt.zero_grad()
        x.grad = None
        l_ = objective()
        l_.backward()
        opt.step()
    assert float(objective()) < l0


def test_batchnorm_on_arrays_of_more_than_two_dimensions(B):
    """InvertibleBatchNorm on (W, H, C, B) / (L, C, B) arrays: channel axis = ndims − 1 (normalise.jl:41-47), the
    log-Jacobian is fill(sum(logs − log(v + eps)/2), B) -- no spatial factor (:66-67) -- both directions."""
    import torch

    rng = np.random.default_rng(321)
    for shape in ((5, 3, 6, 37), (7, 4, 19), (2, 2, 2, 3, 11)):
        C = shape[-2]
        b, logs, m = [(rng.standard_normal(C) * 0.3).astype(f32) for _ in range(3)]
        v = rng.uniform(0.5, 1.5, C).astype(f32)
        bn = B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v)
        obn = O.BatchNormParams(b, logs, m, v, f32(1e-5), f32(0.1))
        x = rng.standard_normal(shape).astype(f32)
        xd = torch.from_numpy(np.asfortranarray(x)).cuda()  # Julia layout: first axis fastest
        assert xd.stride(0) == 1
        y, lj = B.with_logabsdet_jacobian(bn, xd)
        yo, ljo = O.batchnorm_forward(obn, x.astype(np.float64))
        assert tuple(y.shape) == shape and tuple(y.stride()) == tuple(xd.stride()) and lj.shape == (shape[-1],)
        assert rel(y.cpu().numpy(), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL
        assert np.array_equal(B.transform(bn, xd).cpu().numpy(), y.cpu().numpy())
        assert np.array_equal(B.to_numpy(B.logabsdetjac(bn, xd)), B.to_numpy(lj))
        xi, lji = B.with_logabsdet_jacobian(B.inverse(bn), y)
        xo, ljio = O.batchnorm_inverse(obn, y.cpu().numpy().astype(np.float64))
        assert rel(xi.cpu().numpy(), xo) <= RTOL and rel(B.to_numpy(lji), ljio) <= RTOL
        with pytest.raises(RuntimeError, match="expected"):
            B.with_logabsdet_jacobian(B.InvertibleBatchNorm(C + 1), xd)
    with pytest.raises(ValueError):  # row-major (not Julia-layout) array
        B.with_logabsdet_jacobian(bn, torch.zeros((2, 2, 2, 3, 11), device="cuda"))


def test_realnvp_trains_through_autograd(B):
    """BASELINE config 5's flow structure as a torch module on the device path: gradients of the NLL w.r.t. every
    parameter equal the oracle's layer-by-layer VJP chain, and a few SGD steps lower the objective."""
    import torch

    torch.manual_seed(0)
    D, N, nb = 64, 2048, 3
    flow = B.autograd.RealNVP(D, nb, scale=0.1)  # (scale 0.5 makes exp(-s) overflow fp32 after three blocks)
    with torch.no_grad():
        for p_ in list(flow.c) + list(flow.b) + list(flow.logs):
            p_.add_(0.05 * torch.randn_like(p_))
    y = (torch.randn((N, D), device="cuda") * 1.3 + 0.2).t()
    loss = flow.nll(y)
    loss.backward()
    # oracle: the same objective differentiated layer by layer in float64
    yo = y.cpu().numpy().astype(np.float64)
    acts, cur = [], yo
    order = []
    for l in reversed(range(nb)):
        obn = O.BatchNormParams(*[t.detach().cpu().numpy().astype(np.float64) for t in (flow.b[l], flow.logs[l], flow.m[l], flow.v[l])],
                                np.float64(np.float32(1e-5)), np.float64(0.1))
        order.append(("bn", l, obn, cur))
        cur, _ = O.batchnorm_inverse(obn, cur)
        m_ = flow.masks[l]
        Wl, cl_ = flow.W[l].detach().cpu().numpy().astype(np.float64), flow.c[l].detach().cpu().numpy().astype(np.float64)
        order.append(("cpl", l, (m_.indices_1, m_.indices_2, Wl, cl_), cur))
        cur, _ = O.coupling_affine_inverse(m_.indices_1, m_.indices_2, Wl, cl_, cur)
    xbar = cur.copy()            # d(nll)/dx = x   (nll = −Σ(−½‖x‖² + lj) + const)
    ljbar = -np.ones(N)
    grads = {}
    for kind, l, prm, inp in reversed(order):
        if kind == "cpl":
            xbar, Wb, cb = O.coupling_affine_vjp(prm[0], prm[1], prm[2], prm[3], inp, xbar, ljbar, inverse=True)
            grads[("W", l)], grads[("c", l)] = Wb, cb
        else:
            xbar, bb, lb = O.batchnorm_eval_vjp(prm, inp, xbar, ljbar, inverse=True)
            grads[("b", l)], grads[("logs", l)] = bb, lb
    for l in range(nb):
        for name, par in (("W", flow.W[l]), ("c", flow.c[l]), ("b", flow.b[l]), ("logs", flow.logs[l])):
            assert rel(par.grad.cpu().numpy(), grads[(name, l)]) <= 5e-5, (name, l, rel(par.grad.cpu().numpy(), grads[(name, l)]))
    opt = torch.optim.SGD(flow.parameters(), lr=1e-6)
    l0 = float(loss)
    for _ in range(15):
        opt.zero_grad()
        lo = flow.nll(y)
        lo.backward()
        opt.step()
    assert float(flow.nll(y)) < l0


@pytest.mark.parametrize("D,flags", [(64, (True,) * 6), (32, (True, False, True)), (128, (False, True, True, False)), (10, (True, True))])
def test_radial_chain_vjp_inverse_and_mixed_directions(B, D, flags):
    """Reverse mode through Inverse(RadialLayer) (compute_r by the implicit-function rule) and through chains that mix
    directions, against the finite-difference-pinned float64 oracle (radial_chain_vjp_dir)."""
    import torch

    rng = np.random.default_rng(300 + D + len(flags))
    N = 1777
    pairs = [make_case("radial", D, rng) for _ in flags]
    chain = B.Composed(*[(B.inverse(p[0]) if f else p[0]) for p, f in zip(pairs, flags)])
    x, ybar, ljbar = rng.standard_normal((D, N)).astype(f32), rng.standard_normal((D, N)).astype(f32), rng.standard_normal(N).astype(f32)
    xbar, grads = B.radial_chain_vjp(chain, B.from_numpy(x), B.from_numpy(ybar), torch.as_tensor(ljbar, device="cuda"))
    oparams = [(p[1].params["alpha_raw"].astype(np.float64), p[1].params["beta"].astype(np.float64), p[1].params["z0"].astype(np.float64)) for p in pairs]
    xo, go = O.radial_chain_vjp_dir(oparams, flags, x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64))
    assert rel(B.to_numpy(xbar), xo) <= RTOL, rel(B.to_numpy(xbar), xo)
    for g, (ao, bo, zo) in zip(grads, go):
        sc = np.sqrt(N)  # sums of N O(1) terms
        assert abs(float(g["α_"]) - float(ao)) <= 5e-5 * max(abs(float(ao)), sc), (float(g["α_"]), float(ao))
        assert abs(float(g["β"]) - float(bo)) <= 5e-5 * max(abs(float(bo)), sc), (float(g["β"]), float(bo))
        assert rel(B.to_numpy(g["z_0"]), zo) <= 5e-5, rel(B.to_numpy(g["z_0"]), zo)
    # the NLL path of a radial flow through autograd: gradients flow, the loss decreases
    if D == 64:
        torch.manual_seed(1)
        flow = B.autograd.RadialFlow(D, 3)
        y = torch.randn((N, D), device="cuda").t()

        def nll():
            xx, lj = flow.inverse(y)
            return -((-0.5 * (xx * xx).sum(0)) + lj).sum()

        l0 = nll()
        l0.backward()
        assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in flow.parameters())
        opt = torch.optim.SGD(flow.parameters(), lr=1e-5)
        for _ in range(10):
            opt.zero_grad()
            lo = nll()
            lo.backward()
            opt.step()
        assert float(nll()) < float(l0)
