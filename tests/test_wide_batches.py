"""Wide batches (256 < D <= 1024, Float64 up to 2048): the kernel instantiations that only run past D = 256 -- the
lane-group kernel's <32,4,2> / <32,8,1> builds, chains split at the shared-memory budget, coupling layers with hundreds of
pass-through rows, the 1024-thread elementwise VJP, the wide BatchNorm VJP builds -- against the float64 oracle within the
parity gate of test_gpu_parity, and the documented limits of include/b2b.h on both sides."""
import zlib

import numpy as np
import pytest

from oracle import oracle_np as O
from test_chain_vjp import check_chain, stacked_case
from test_gpu_parity import gate, make_case, rel

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5
EUNSUPPORTED = -2  # B2B_EUNSUPPORTED of include/b2b.h


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def _seed(*key):
    return np.random.default_rng(zlib.crc32("-".join(map(str, key)).encode()))


def _launches(B):
    return B.lib().b2b_last_launch_count()


def _raises(B, status, fn):
    with pytest.raises(B.B2BError) as ei:
        fn()
    assert ei.value.status == status, ei.value.status


# ---- 1. single layers: strides, misaligned pointers, in place, accumulation, logjac-only ----------------------------------
WIDE_KINDS = ["planar", "radial", "batchnorm", "permute", "stacked", "bounded", "leaky_relu", "rqs", "coupling"]


@pytest.mark.parametrize("D", [257, 260, 512, 513, 1000, 1024])
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_wide_layer_layouts_in_place_and_accumulation(B, kind, D):
    """Every layout of the batch gives the bit-identical result of the contiguous call: a padded column stride and a
    base pointer one float off the 16-byte boundary (the scalar-load build), in place, logjac only."""
    import torch

    rng = _seed("layout", kind, D)
    lay, olay = make_case(kind, D, rng)
    N = 4097
    x = (rng.uniform(-0.9, 2.9, (D, N)) if kind == "bounded" else rng.standard_normal((D, N))).astype(f32)
    y, lj = B.with_logabsdet_jacobian(lay, B.from_numpy(x))
    ref_launches = _launches(B)
    yh, ljh = B.to_numpy(y), B.to_numpy(lj)
    yo, ljo = olay.forward(x.astype(np.float64))
    if kind == "permute":
        assert np.array_equal(yh.view(np.uint32), olay.forward(x)[0].view(np.uint32)) and np.all(ljh == 0)
    else:
        assert rel(yh, yo) <= RTOL and rel(ljh, ljo) <= gate(olay.forward(x)[1], ljo), (rel(yh, yo), rel(ljh, ljo))
    # fused column-local layers: one launch; coupling: W image + tensor-core kernel + the 1-column ragged tail, or the
    # exact-fp32 kernel alone where the mask's x₂ rows do not start on a 16-byte boundary
    assert ref_launches in ((1, 3) if kind == "coupling" else (1,)), ref_launches
    # the tensor-core coupling path needs 16-byte aligned columns: other layouts run the exact-fp32 kernel (same gate)
    same = torch.equal if kind != "coupling" else (lambda a, b: rel(B.to_numpy(a), B.to_numpy(b)) <= 2e-5)
    # padded column stride (ld = D + 1) into a padded output; the padding stays untouched
    buf = torch.zeros((N, D + 1), device="cuda")
    xv = buf[:, :D].t()
    xv.copy_(B.from_numpy(x))
    obuf = torch.full((N, D + 3), 7.0, device="cuda")
    yv = obuf[:, :D].t()
    _, ljv = B.run_chain(lay, xv, y=yv)
    assert same(yv, y) and same(ljv, lj) and bool((obuf[:, D:] == 7.0).all())
    # base pointer one float off the 16-byte boundary
    flat = torch.zeros(D * N + 1, device="cuda")
    xm = flat[1:].view(N, D).t()
    xm.copy_(B.from_numpy(x))
    y2, lj2 = B.with_logabsdet_jacobian(lay, xm)
    assert same(y2, y) and same(lj2, lj)
    # logjac only (no D x N store)
    assert torch.equal(B.logabsdetjac(lay, xm), lj2)
    assert torch.equal(B.logabsdetjac(lay, B.from_numpy(x)), lj)
    # in place, accumulating into an existing logjac
    xi = B.from_numpy(x)
    acc = torch.full((N,), 0.25, device="cuda")
    B.with_logabsdet_jacobian_(lay, xi, None, acc)
    assert torch.equal(xi, y)
    assert float((acc - 0.25 - lj).abs().max()) <= 1e-6 * max(1.0, float(lj.abs().max()))


# ---- 2. chains split at the shared-memory budget -------------------------------------------------------------------------
def _planar_bn_flow(B, D, rng, L=8):
    dev, ol = [], []
    for _ in range(L):
        p, op = make_case("planar", D, rng)
        b, ob = make_case("batchnorm", D, rng)
        dev += [p, b]
        ol += [op, ob]
    return dev, ol


@pytest.mark.parametrize("D", [512, 1024])
def test_planar_batchnorm_flow_logpdf(B, D):
    """logpdf of inverse(8 x (PlanarLayer ∘ InvertibleBatchNorm)) + MvNormal: at D = 1024 the staged parameters of the
    17-layer run exceed one kernel's shared memory, so the run is split; the result is the layer-by-layer one."""
    import torch

    rng = _seed("pbn", D)
    N = 3001
    dev, ol = _planar_bn_flow(B, D, rng)
    flow = B.Composed(*dev)
    mu, sigma = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 2.0, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu, sigma), B.inverse(flow))
    y = rng.standard_normal((D, N)).astype(f32)
    yd = B.from_numpy(y)
    # logpdf(td, y) runs flow itself on y (inverse of the inverse), then the base density
    lp = B.to_numpy(B.logpdf(td, yd))
    # 17 layers: one launch at D = 512; at D = 1024 their 205 072 B of staged parameters take two
    assert (_launches(B) >= 2) == (D == 1024), _launches(B)
    xo, ljo = O.chain_forward(ol, y.astype(np.float64))
    lpo = O.mvnormal_diag_logpdf(mu.astype(np.float64), sigma.astype(np.float64), xo) + ljo
    xo32, ljo32 = O.chain_forward(ol, y)
    lpo32 = O.mvnormal_diag_logpdf(mu, sigma, xo32) + ljo32
    assert rel(lp, lpo) <= gate(lpo32, lpo), (rel(lp, lpo), rel(lpo32, lpo))
    tot, lp2 = B.logpdf_sum(td, yd)
    assert np.array_equal(B.to_numpy(lp2), lp)
    assert abs(float(tot) - float(lp.astype(np.float64).sum())) <= 1e-9 * abs(float(tot)) + 1e-6
    # layer by layer: the same numbers as the split run
    buf = B.from_numpy(y)
    acc = torch.zeros(N, dtype=torch.float32, device="cuda")
    for lay in dev:
        buf, acc = B.with_logabsdet_jacobian_(lay, buf, None, acc)
    base = B.to_numpy(B.logpdf(B.MvNormal(D, mu, sigma), buf))
    assert rel(lp, base + B.to_numpy(acc)) <= 2e-6
    # the forward chain (16 layers, one launch at both D): y and logjac, and the logjac-only call
    x1, lj1 = B.with_logabsdet_jacobian(flow, yd)
    assert rel(B.to_numpy(x1), B.to_numpy(buf)) <= 2e-6 and rel(B.to_numpy(lj1), B.to_numpy(acc)) <= 2e-6
    assert torch.equal(B.logabsdetjac(flow, yd), lj1)


def test_host_pipeline_logpdf_of_a_split_chain(B):
    """The host-buffer pipeline runs a logpdf that needs two launches per chunk (D = 1024, the 17-layer chain of
    test_planar_batchnorm_flow_logpdf) without a D x N output: its staging buffer carries the intermediate.  Two chunks of
    columns; the result is the device path's, bit for bit."""
    import torch

    rng = _seed("hostpbn")
    D, N = 1024, (1 << 16) + 1001
    dev, _ = _planar_bn_flow(B, D, rng)
    mu, sigma = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 2.0, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu, sigma), B.inverse(B.Composed(*dev)))
    yh = B.from_numpy(rng.standard_normal((D, N)).astype(f32), device="cpu", pin_memory=True)
    yd = yh.cuda()
    lp_h = B.logpdf(td, yh)
    assert not lp_h.is_cuda
    lp_d = B.logpdf(td, yd)
    assert torch.equal(lp_h, lp_d.cpu())
    tot_h, _ = B.logpdf_sum(td, yh)
    tot_d, _ = B.logpdf_sum(td, yd)
    assert abs(float(tot_h) - float(tot_d)) <= 1e-9 * abs(float(tot_d))


def test_split_chain_workspace_and_launches(B):
    """The workspace query plans the same segments as the call: a split logjac-only chain gets its D x N scratch, and a
    chain that fits one kernel is still one launch."""
    from bijectors_jl_b200.interface import _desc_array

    rng = _seed("ws")
    D, N = 1024, 100
    dev, _ = _planar_bn_flow(B, D, rng, L=10)  # 20 layers: 240 KB of staged parameters
    descs = B.Composed(*dev)._descs(False, D)
    arr = _desc_array(descs)
    L_ = B.lib()
    with_y = L_.b2b_chain_workspace_bytes(arr, len(descs), D, N, 1, 0)
    no_y = L_.b2b_chain_workspace_bytes(arr, len(descs), D, N, 0, 0)
    assert no_y >= with_y + D * N * 4
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    B.with_logabsdet_jacobian(B.Composed(*dev), x)
    assert _launches(B) >= 2
    B.with_logabsdet_jacobian(B.Composed(*dev[:4]), x)
    assert _launches(B) == 1


# ---- 3. coupling layers at wide D --------------------------------------------------------------------------------------
def _coupling(B, D, idx1, idx2, rng, scale=0.2):
    n1, n2 = len(idx1), len(idx2)
    W = (rng.standard_normal((2 * n1, n2)) * scale / np.sqrt(n2)).astype(f32)
    c = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    return (B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2)),
            O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c)))


def _mask(D, kind, rng, n=128):
    if kind == "halves":  # contiguous 128-row halves, D - 256 pass-through rows after them
        return list(range(1, n + 1)), list(range(n + 1, 2 * n + 1))
    if kind == "tail":  # contiguous, x₂ before x₁ at the end of the column
        return list(range(D - n + 1, D + 1)), list(range(D - 2 * n + 1, D - n + 1))
    rows = (rng.permutation(D) + 1).tolist()
    return sorted(rows[:n]), sorted(rows[n:2 * n])


@pytest.mark.parametrize("N", [4096, 4097])
@pytest.mark.parametrize("D,mask", [(1000, "halves"), (1000, "tail"), (1024, "halves"), (512, "scattered"),
                                    (747, "scattered"), (1000, "scattered")])
def test_wide_coupling(B, D, mask, N):
    """Affine coupling with hundreds of pass-through rows: works for every N (the ragged tail of the tensor-core path runs
    the exact-fp32 kernel), both kernels match the oracle, x₂ / x₃ rows are bit-exact, in place and inverse."""
    import torch

    rng = _seed("cpl", D, mask, N)
    idx1, idx2 = _mask(D, mask, rng)
    cl, ol = _coupling(B, D, idx1, idx2, rng)
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)
    y, lj = B.with_logabsdet_jacobian(cl, xd)
    yo, ljo = ol.forward(x.astype(np.float64))
    assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL, (rel(B.to_numpy(y), yo), rel(B.to_numpy(lj), ljo))
    keep = np.setdiff1d(np.arange(D), np.asarray(idx1) - 1)
    assert np.array_equal(B.to_numpy(y)[keep], x[keep])
    B.lib().b2b_set_kernel_variant(10)  # the exact-fp32 CUDA-core kernel on the whole batch
    try:
        y2, lj2 = B.with_logabsdet_jacobian(cl, xd)
        assert _launches(B) == 1
        assert torch.equal(B.logabsdetjac(cl, xd), lj2)
    finally:
        B.lib().b2b_set_kernel_variant(0)
    assert rel(B.to_numpy(y2), yo) <= RTOL and rel(B.to_numpy(lj2), ljo) <= RTOL
    assert np.array_equal(B.to_numpy(y2)[keep], x[keep])
    # inverse in place, accumulating: back to x and a zero total log-Jacobian
    yi = y2.clone()
    acc = lj2.clone()
    B.with_logabsdet_jacobian_(B.inverse(cl), yi, None, acc)
    xo, _ = ol.inverse(B.to_numpy(y2).astype(np.float64))
    assert rel(B.to_numpy(yi), xo) <= gate(ol.inverse(B.to_numpy(y2))[0], xo)
    assert float(acc.abs().max()) <= 1e-4 * max(1.0, float(np.abs(ljo).max()))
    assert np.array_equal(B.to_numpy(yi)[keep], x[keep])


@pytest.mark.parametrize("D,mask", [(1000, "halves"), (1021, "tail"), (768, "scattered")])
def test_wide_coupling_with_folded_batchnorm(B, D, mask):
    """BatchNorm neighbours folded into the coupling launch apply to the pass-through rows too (out of place and in
    place), with the tensor-core kernel, the exact-fp32 kernel and without folding."""
    import torch

    rng = _seed("fold", D, mask)
    N = 2049
    idx1, idx2 = _mask(D, mask, rng)
    cl, ol = _coupling(B, D, idx1, idx2, rng)
    b1, ob1 = make_case("batchnorm", D, rng)
    b2, ob2 = make_case("batchnorm", D, rng)
    flow = B.Composed(b1, cl, b2)
    olayers = [ob1, ol, ob2]
    x = rng.standard_normal((D, N)).astype(f32)
    xd = B.from_numpy(x)
    yo, ljo = O.chain_forward(olayers, x.astype(np.float64))
    outs = []
    for variant in (0, 10, 100):
        B.lib().b2b_set_kernel_variant(variant)
        try:
            y, lj = B.with_logabsdet_jacobian(flow, xd)
            xi = B.from_numpy(x)
            B.with_logabsdet_jacobian_(flow, xi)
        finally:
            B.lib().b2b_set_kernel_variant(0)
        assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= RTOL, (variant, rel(B.to_numpy(y), yo))
        assert torch.equal(xi, y), variant
        outs.append(y)
    xo, ljio = O.chain_inverse(olayers, B.to_numpy(outs[0]).astype(np.float64))
    xi, lji = B.with_logabsdet_jacobian(B.inverse(flow), outs[0])
    assert rel(B.to_numpy(xi), xo) <= RTOL and rel(B.to_numpy(lji), ljio) <= RTOL


# ---- 4. reverse mode ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [257, 1000, 1024])
def test_elementwise_run_with_mvnormal_vjp(B, D):
    """Eight Stacked / Permute layers and the terminal MvNormal with μ̄ and σ̄: one launch of the 1024-thread
    elementwise VJP kernel at its largest shared-memory size."""
    rng = _seed("ew", D)
    N = 777
    st = [stacked_case(B, names, D) for names in (["logit", "shift"], ["scale", "leaky_relu"], ["shift", "scale"],
                                                   ["leaky_relu", "identity"], ["scale", "shift"])]
    perms = [(rng.permutation(D) + 1).tolist() for _ in range(3)]
    P = [(B.Permute(p), O.Layer("permute", dict(A=O.permute_matrix_from_indices(p)))) for p in perms]
    order = [st[0], P[0], st[1], P[1], st[2], P[2], st[3], st[4]]
    flow = B.inverse(B.Composed(*[d for d, _ in order]))  # logpdf runs the composed chain itself
    olayers = [o for _, o in order]
    mu, sigma = (rng.standard_normal(D) * 0.3).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    base = B.MvNormal(D, mu=mu, sigma=sigma)
    x = rng.standard_normal((D, N))
    x[: D // 2] = rng.uniform(-0.9, 2.9, (D // 2, N))  # the Logit rows of the first layer
    check_chain(B, flow, olayers, [False] * 8, x, None, rng.standard_normal(N), mu, sigma, base, terminal=True)


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D", [257, 512, 513, 768, 769, 1000, 1024])
def test_wide_batchnorm_eval_vjp(B, D, inv):
    rng = _seed("bnvjp", D, inv)
    N = 1025
    lay, olay = make_case("batchnorm", D, rng)
    x = rng.standard_normal((D, N))
    check_chain(B, B.inverse(lay) if inv else lay, [olay], [inv], x, rng.standard_normal((D, N)), rng.standard_normal(N))


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("D,mask", [(512, "scattered"), (747, "scattered"), (747, "tail")])
def test_wide_coupling_vjp(B, D, mask, inv):
    """n1 = n2 = 128 (the float4 kernel) at D up to its shared-memory limit of 747 rows."""
    rng = _seed("cplvjp", D, mask, inv)
    N = 1100
    idx1, idx2 = _mask(D, mask, rng)
    cl, ol = _coupling(B, D, idx1, idx2, rng, scale=0.1)
    x = rng.standard_normal((D, N))
    check_chain(B, B.inverse(cl) if inv else cl, [ol], [inv], x, rng.standard_normal((D, N)), rng.standard_normal(N))


def test_wide_chain_logpdf_vjp_every_parameter(B):
    """chain_vjp and logpdf_vjp through BatchNorm, Stacked, Permute, Coupling and MvNormal at D = 512: every parameter
    cotangent against the oracle."""
    rng = _seed("chain512")
    D, N = 512, 1300
    bn1, obn1 = make_case("batchnorm", D, rng)
    st, ost = stacked_case(B, ["shift", "scale", "leaky_relu"], D)
    perm = (rng.permutation(D) + 1).tolist()
    idx1, idx2 = _mask(D, "scattered", rng)
    cl, ocl = _coupling(B, D, idx1, idx2, rng, scale=0.1)
    bn2, obn2 = make_case("batchnorm", D, rng)
    dev = [bn1, st, B.Permute(perm), cl, bn2]
    ol = [obn1, ost, O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))), ocl, obn2]
    x = rng.standard_normal((D, N))
    check_chain(B, B.Composed(*dev), ol, [False] * 5, x, rng.standard_normal((D, N)), rng.standard_normal(N))
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.4, D).astype(f32)
    check_chain(B, B.inverse(B.Composed(*dev)), ol, [False] * 5, x, None, rng.standard_normal(N), mu, sigma,
                B.MvNormal(D, mu=mu, sigma=sigma), terminal=True)


# ---- 5. sampling ---------------------------------------------------------------------------------------------------------
def test_chain_sample_two_pass_at_d1000(B):
    """b2b_chain_sample_f32 at D = 1000 (base samples first, then the chain in place) is the oracle's stream pushed
    through the oracle's chain."""
    rng = _seed("sample1000")
    D, n = 1000, 1500
    seed, off = 0xDEAD_BEEF_1234, 3
    mu, sigma = (rng.standard_normal(D) * 0.3).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    pairs = [make_case(k, D, rng) for k in ("planar", "stacked", "rqs", "coupling", "batchnorm", "radial")]
    td = B.transformed(B.MvNormal(D, mu, sigma), B.Composed(*[p[0] for p in pairs]))
    y, lj = B.rand(td, n, seed=seed, offset=off, with_logjac=True)
    zo = O.philox_normals(seed, off, D, n, mu=mu.astype(np.float64), sigma=sigma.astype(np.float64))
    olayers = [p[1] for p in pairs]
    yo, ljo = O.chain_forward(olayers, zo)
    yo32, ljo32 = O.chain_forward(olayers, zo.astype(f32))
    assert rel(B.to_numpy(y), yo) <= gate(yo32, yo) and rel(B.to_numpy(lj), ljo) <= gate(ljo32, ljo), (rel(B.to_numpy(y), yo), rel(B.to_numpy(lj), ljo))


# ---- 6. the documented limits, on both sides ------------------------------------------------------------------------------
def _sentinel_call(B, fn, *bufs, f32=True):
    """fn() must fail with B2B_EUNSUPPORTED before launching anything: every buffer bit-identical and (Float32 chains,
    which b2b_last_launch_count reports on) no launch counted."""
    import torch

    before = [b.clone() for b in bufs]
    _raises(B, EUNSUPPORTED, fn)
    if f32:
        assert _launches(B) == 0
    torch.cuda.synchronize()
    for a, b in zip(before, bufs):  # bit patterns: the sentinels are NaN
        bits = torch.int64 if a.dtype == torch.float64 else torch.int32
        assert torch.equal(a.view(bits), b.view(bits))


def test_float64_limit(B):
    import torch

    rng = _seed("f64lim")
    for D, ok in ((2048, True), (2049, False)):
        lay = B.PlanarLayer(rng.standard_normal(D) / np.sqrt(D), rng.standard_normal(D) / np.sqrt(D), rng.standard_normal(1),
                            dtype=torch.float64)
        x = B.from_numpy(rng.standard_normal((D, 9)), dtype=np.float64)
        y = torch.full((9, D), float("nan"), dtype=torch.float64, device="cuda").t()
        lj = torch.full((9,), -3.0, dtype=torch.float64, device="cuda")
        if ok:
            B.run_chain(lay, x, y=y, logjac=lj)
            o = O.Layer("planar", dict(w=B.to_numpy(lay.w), u=B.to_numpy(lay.u), b=B.to_numpy(lay.b)))
            yo, ljo = o.forward(B.to_numpy(x))
            assert rel(B.to_numpy(y), yo) <= 1e-12 and rel(B.to_numpy(lj), ljo) <= 1e-12
        else:
            _sentinel_call(B, lambda: B.run_chain(lay, x, y=y, logjac=lj), y, lj, f32=False)


def test_batchnorm_training_limit(B):
    import torch

    rng = _seed("bntrain")
    D, N = 1025, 300
    bn = B.InvertibleBatchNorm(D, training=True)
    m0, v0 = bn.m.clone(), bn.v.clone()
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    _raises(B, EUNSUPPORTED, lambda: bn.train_forward(x))
    torch.cuda.synchronize()
    assert torch.equal(bn.m, m0) and torch.equal(bn.v, v0)


@pytest.mark.parametrize("D,K1,ok", [(512, 8, True), (512, 9, False), (1024, 4, True), (1024, 5, False), (257, 9, False)])
def test_rqs_knot_limit_by_d(B, D, K1, ok):
    """RQS knot tables in the fused kernels: K1 <= 8 up to D = 512, K1 <= 4 up to D = 1024.  Past the limit nothing is
    launched -- also when the RQS layer comes after a coupling layer that could have run on its own."""
    import torch

    rng = _seed("rqslim", D, K1)
    K = K1 - 1
    spl = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                    rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    W, H, Dv = spl.knots()
    osp = O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv))
    N = 300
    x = (rng.standard_normal((D, N)) * 1.5).astype(f32)
    xd = B.from_numpy(x)
    y = torch.full((N, D), float("nan"), device="cuda").t()
    lj = torch.full((N,), -3.0, device="cuda")
    if ok:
        B.run_chain(spl, xd, y=y, logjac=lj)
        yo, ljo = osp.forward(x.astype(np.float64))
        assert rel(B.to_numpy(y), yo) <= RTOL and rel(B.to_numpy(lj), ljo) <= gate(osp.forward(x)[1], ljo)
        return
    _sentinel_call(B, lambda: B.run_chain(spl, xd, y=y, logjac=lj), y, lj)
    idx1, idx2 = _mask(D, "halves", rng)
    cl, _ = _coupling(B, D, idx1, idx2, rng)
    _sentinel_call(B, lambda: B.run_chain(B.Composed(cl, B.PlanarLayer(D), spl), xd, y=y, logjac=lj), y, lj)


@pytest.mark.parametrize("D,ok", [(747, True), (748, False), (760, False)])
@pytest.mark.parametrize("chain", ["coupling", "batchnorm_coupling"])
def test_coupling_vjp_limit_query_matches_call(B, D, ok, chain):
    """b2b_chain_vjp_workspace_bytes returns 0 exactly when b2b_chain_vjp_f32 refuses the chain, and a refused chain
    launches nothing (not even the forward recompute of the segments before the coupling)."""
    from bijectors_jl_b200.interface import _desc_array

    rng = _seed("cvlim", D, chain)
    N = 300
    idx1, idx2 = _mask(D, "halves", rng)
    cl, ocl = _coupling(B, D, idx1, idx2, rng, scale=0.1)
    bn, obn = make_case("batchnorm", D, rng)
    dev, ol = ([cl], [ocl]) if chain == "coupling" else ([bn, cl], [obn, ocl])
    descs = B.Composed(*dev)._descs(False, D)
    arr = _desc_array(descs)
    L_ = B.lib()
    need = L_.b2b_chain_vjp_workspace_bytes(arr, len(descs), D, N)
    x = rng.standard_normal((D, N))
    if ok:
        assert need > 0
        check_chain(B, B.Composed(*dev), ol, [False] * len(dev), x, rng.standard_normal((D, N)), rng.standard_normal(N))
        return
    assert need == 0
    _vjp_refused(B, arr, len(descs), x, D, N)


def _vjp_refused(B, arr, L, x, D, N):
    """b2b_chain_vjp_f32 refuses the chain with B2B_EUNSUPPORTED, launches nothing and leaves x̄ untouched."""
    import torch

    from bijectors_jl_b200.interface import _stream

    xd = B.from_numpy(x.astype(f32))
    xb = torch.full((N, D), float("nan"), device="cuda").t()
    ws = torch.empty((1 << 20,), dtype=torch.uint8, device="cuda")
    before = xb.clone()
    rc = B.lib().b2b_chain_vjp_f32(arr, L, xd.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, ws.data_ptr(),
                                   ws.numel(), _stream())
    assert rc == EUNSUPPORTED, rc
    assert _launches(B) == 0
    torch.cuda.synchronize()
    assert torch.equal(xb.view(torch.int32), before.view(torch.int32))


@pytest.mark.parametrize("K1,ok", [(17, True), (18, False)])
def test_chain_vjp_query_matches_call_through_the_forward_recompute(B, K1, ok):
    """The reverse mode recomputes the forward of every segment but the last: an RQS layer the fused forward kernels
    cannot stage (K1 > 17 at D = 256) makes the workspace query return 0 and the call refuse the chain up front, although
    the RQS reverse-mode kernel itself would take it."""
    from bijectors_jl_b200.interface import _desc_array

    rng = _seed("vjpfwd", K1)
    D, N, K = 256, 400, K1 - 1
    bn, obn = make_case("batchnorm", D, rng)
    spl = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                    rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    W, H, Dv = spl.knots()
    st, ost = stacked_case(B, ["shift", "scale"], D)
    dev, ol = [bn, spl, st], [obn, O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv)), ost]
    descs = B.Composed(*dev)._descs(False, D)
    arr = _desc_array(descs)
    need = B.lib().b2b_chain_vjp_workspace_bytes(arr, len(descs), D, N)
    x = rng.standard_normal((D, N)) * 1.5
    if ok:
        assert need > 0
        check_chain(B, B.Composed(*dev), ol, [False] * 3, x, rng.standard_normal((D, N)), rng.standard_normal(N))
        return
    assert need == 0
    _vjp_refused(B, arr, len(descs), x, D, N)
