"""Reparameterised sampling on the device: rand_logpdf (b2b_chain_sample_logq_f32), rand_vjp (b2b_chain_sample_vjp_f32)
and autograd.Flow.rsample against the float64 reference of tests/rsample_oracle.py on the same Philox draw."""
import ctypes

import numpy as np
import pytest

import coupling_deep_mlp_oracle as DM
import coupling_deep_mlp_rqs_oracle as DR
import coupling_mlp_oracle as M
import coupling_mlp_rqs_oracle as MR
import mvnormal_tril_oracle as T
import rsample_oracle as R
import scale_matrix_oracle as SM
import spline_coupling_oracle as SC
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

f32 = np.float32
RTOL = 1e-5
SEED = 0x5EED1234ABCD


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def planar(B, D, rng, scale=0.3):
    w, u = (rng.standard_normal(D) * scale / np.sqrt(D) * 4).astype(f32), (rng.standard_normal(D) * scale).astype(f32)
    b = rng.standard_normal(1).astype(f32)
    return B.PlanarLayer(w, u, b), O.Layer("planar", dict(w=w, u=u, b=b))


def rqs(B, D, rng, K=6):
    spl = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                    rng.standard_normal((D, K - 1)).astype(f32), 3.0)
    W, H, Dv = spl.knots()
    return spl, O.Layer("rqs", dict(widths=W, heights=H, derivs=Dv))


def permute(B, D, rng):
    perm = (rng.permutation(D) + 1).tolist()
    return B.Permute(perm), O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm)))


def stacked(B, D):
    half = D // 2
    return (B.Stacked([B.Shift(0.7), B.Scale(-1.3)], [(1, half), (half + 1, D)]),
            O.Layer("stacked", dict(ops=[(O.EW.SHIFT, f32(0.7)), (O.EW.SCALE, f32(-1.3))], ranges=[(1, half), (half + 1, D)])))


def coupling(B, D, rng):
    n1 = D // 2
    W = (rng.standard_normal((2 * n1, D - n1)) * 0.05).astype(f32)
    c = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
    idx1, idx2 = list(range(1, n1 + 1)), list(range(n1 + 1, D + 1))
    return (B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2)),
            O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c)))


def make_base(B, D, rng, kind):
    """(device MvNormal, mu, sigma, L) for kind in {"std", "diag", "tril"}."""
    if kind == "std":
        return B.MvNormal(D), None, None, None
    mu = (rng.standard_normal(D) * 0.3).astype(f32)
    if kind == "diag":
        sigma = rng.uniform(0.6, 1.4, D).astype(f32)
        return B.MvNormal(D, mu=mu, sigma=sigma), mu, sigma, None
    L = T.random_tril(rng, D).astype(f32)
    return B.MvNormal(D, mu=mu, scale_tril=L), mu, None, L


def _rows(rng, D, n1, n2):
    rows = rng.permutation(D) + 1
    return [int(i) for i in rows[:n1]], [int(i) for i in rows[n1:n1 + n2]]


def kind_layer(B, D, rng, kind):
    """(device layer, oracle layer) of one layer of `kind`, parameters scaled so that every layer's values stay O(1)."""
    if kind == "planar":
        return planar(B, D, rng)
    if kind == "radial":
        a, be = rng.standard_normal(1).astype(f32), rng.standard_normal(1).astype(f32)
        z0 = (rng.standard_normal(D) * 0.1).astype(f32)
        return B.RadialLayer(a, be, z0), O.Layer("radial", dict(alpha_raw=a, beta=be, z0=z0))
    if kind == "rqs":
        return rqs(B, D, rng)
    if kind == "bn":
        b, logs, m = ((rng.standard_normal(D) * 0.1).astype(f32) for _ in range(3))
        v = rng.uniform(0.5, 1.5, D).astype(f32)
        return (B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v),
                O.Layer("batchnorm", dict(bn=O.BatchNormParams(b, logs, m, v, f32(1e-5), f32(0.1)))))
    if kind == "stacked":
        return stacked(B, D)
    if kind == "perm":
        return permute(B, D, rng)
    if kind == "cpl":
        return coupling(B, D, rng)
    if kind == "scale":
        A = SM.well_conditioned(rng, D).astype(f32)
        return B.Scale(A), SM.ScaleLayer(A)
    n1, n2, H, K = D // 4, D - D // 4 - 2, 16, 6
    i1, i2 = _rows(rng, D, n1, n2)
    J = (3 * K - 1) * n1
    if kind == "spl":  # COUPLING_RQS
        W = (rng.standard_normal((J, n2)) * 0.3 / np.sqrt(n2)).astype(f32)
        c = (rng.standard_normal(J) * 0.3).astype(f32)
        return B.Coupling(B.SplineConditioner(W, c, K=K, B=3.0), B.PartitionMask(D, i1, i2)), SC.SplineLayer(i1, i2, W, c, K, 3.0)
    W1 = (rng.standard_normal((H, n2)) * 0.8 / np.sqrt(n2)).astype(f32)
    c1 = (rng.standard_normal(H) * 0.3).astype(f32)
    if kind in ("mlp", "mlp_rqs"):
        rows = 2 * n1 if kind == "mlp" else J
        W2 = (rng.standard_normal((rows, H)) * 0.3 / np.sqrt(H)).astype(f32)
        c2 = (rng.standard_normal(rows) * 0.1).astype(f32)
        if kind == "mlp":
            return (B.Coupling(B.MLPConditioner(W1, c1, W2, c2), B.PartitionMask(D, i1, i2)),
                    M.MLPLayer(i1, i2, W1, c1, W2, c2))
        return (B.Coupling(B.MLPSplineConditioner(W1, c1, W2, c2, K=K, B=3.0), B.PartitionMask(D, i1, i2)),
                MR.MLPSplineLayer(i1, i2, W1, c1, W2, c2, K, 3.0))
    rows = 2 * n1 if kind == "deep_mlp" else J
    weights = [W1, (rng.standard_normal((H, H)) * 1.2 / np.sqrt(H)).astype(f32),
               (rng.standard_normal((rows, H)) * 0.3 / np.sqrt(H)).astype(f32)]
    biases = [c1, (rng.standard_normal(H) * 0.3).astype(f32), (rng.standard_normal(rows) * 0.1).astype(f32)]
    if kind == "deep_mlp":
        return (B.Coupling(B.DeepMLPConditioner(weights, biases), B.PartitionMask(D, i1, i2)),
                DM.DeepMLPLayer(i1, i2, weights, biases))
    if kind == "deep_mlp_rqs":
        return (B.Coupling(B.DeepMLPSplineConditioner(weights, biases, K=K, B=3.0), B.PartitionMask(D, i1, i2)),
                DR.DeepMLPSplineLayer(i1, i2, weights, biases, K, 3.0))
    raise ValueError(kind)


def spec_chain(*spec):
    """A CHAINS entry from (kind, inverse) pairs: each layer is built by kind_layer and inverted when asked."""
    def make(B, D, rng):
        out = []
        for kind, inv in spec:
            d, o = kind_layer(B, D, rng, kind)
            out.append((B.inverse(d) if inv else d, o, inv))
        return out
    return make


def device_z(B, D, N, seed, offset, column_offset):
    """The base draw z the device uses (b2b_randn_f32 with μ = σ = NULL), in float64: both oracles run on the same z."""
    return B.to_numpy(B.MvNormal(D).rand(N, seed=seed, offset=offset, column_offset=column_offset)).astype(np.float64)


CHAINS = {
    "planar8": lambda B, D, rng: [planar(B, D, rng) for _ in range(8)],                     # fused
    "planar_rqs_stacked": lambda B, D, rng: [planar(B, D, rng), rqs(B, D, rng), stacked(B, D), planar(B, D, rng)],
    "permute_coupling": lambda B, D, rng: [planar(B, D, rng), permute(B, D, rng), coupling(B, D, rng)],  # two passes
    "inverse_planar": lambda B, D, rng: [planar(B, D, rng), (B.inverse(planar(B, D, rng)[0]), None)],
    "rqs_stacked": lambda B, D, rng: [stacked(B, D), rqs(B, D, rng, K=4)],  # reverse mode up to D = 256
    "none": lambda B, D, rng: [],
    # the fused kinds besides planar and RQS, through the LOGQ instantiation of the pipeline (radial reverse mode: D <= 128)
    "radial_bn": spec_chain(("radial", 0), ("bn", 0), ("radial", 1), ("bn", 1)),
    # every kind b2b_chain_vjp_f32 accepts, inverse-flagged layers included
    "every_kind": spec_chain(("planar", 0), ("radial", 1), ("rqs", 0), ("bn", 0), ("stacked", 0), ("perm", 0), ("cpl", 0),
                             ("spl", 0), ("scale", 0), ("mlp", 0), ("mlp_rqs", 0), ("deep_mlp", 1), ("deep_mlp_rqs", 0),
                             ("planar", 1), ("cpl", 1), ("scale", 1)),
    "planar_rqs_mlprqs_perm_stacked": spec_chain(("planar", 0), ("rqs", 0), ("mlp_rqs", 0), ("perm", 0), ("stacked", 0)),
    "deep_mlp": spec_chain(("deep_mlp", 0), ("deep_mlp", 1)),
    "permute_rqs": spec_chain(("perm", 0), ("rqs", 0)),  # two passes at D = 256
}
NETWORK = ("every_kind", "planar_rqs_mlprqs_perm_stacked", "deep_mlp")  # gates 4x the float32 reference, as for these kinds
FUSED_D = (32, 64, 128, 256)
# b2b_chain_vjp_f32 takes planar layers up to D = 128, so the sampler refuses planar chains beyond it
CASES = [(c, D) for D in (32, 48, 64, 128) for c in ("planar8", "planar_rqs_stacked", "permute_coupling", "inverse_planar")] + \
    [(c, D) for D in (32, 48, 64, 128, 256) for c in ("rqs_stacked", "none")] + \
    [("radial_bn", D) for D in (32, 48, 64, 128)] + \
    [("every_kind", 64), ("planar_rqs_mlprqs_perm_stacked", 64), ("deep_mlp", 48), ("permute_rqs", 256)]


def build(B, chain, D, rng, base_kind):
    pairs = CHAINS[chain](B, D, rng)
    flags = []
    olayers = []
    dev = []
    for pair in pairs:
        d, o = pair[:2]
        if len(pair) == 3:  # (device layer, oracle layer, inverted)
            olayers.append(o)
            flags.append(bool(pair[2]))
        elif o is None:  # an inverse-flagged planar layer: its oracle is the same layer applied inverted
            lay = d.orig
            olayers.append(O.Layer("planar", dict(w=B.to_numpy(lay.w), u=B.to_numpy(lay.u), b=B.to_numpy(lay.b))))
            flags.append(True)
        else:
            olayers.append(o)
            flags.append(False)
        dev.append(d)
    base, mu, sigma, L = make_base(B, D, rng, base_kind)
    flow = B.Composed(*dev) if dev else None
    td = B.transformed(base, flow) if flow is not None else base
    return td, olayers, flags, mu, sigma, L


# ---- 1. same samples, 2. correct log q, 3. one launch -------------------------------------------------------------------
@pytest.mark.parametrize("chain,D", CASES)
@pytest.mark.parametrize("base_kind", ["std", "diag", "tril"])
def test_samples_and_logq(B, base_kind, chain, D):
    rng = np.random.default_rng(D * 7 + len(chain) + len(base_kind))
    N, off, col = 3001, 3, 17
    td, ol, flags, mu, sigma, L = build(B, chain, D, rng, base_kind)
    y, lq = B.rand_logpdf(td, N, seed=SEED, offset=off, column_offset=col)
    launches = B.lib().b2b_last_launch_count()
    y1, lj = B.rand(td, N, seed=SEED, offset=off, column_offset=col, with_logjac=True)
    y0 = B.rand(td, N, seed=SEED, offset=off, column_offset=col)
    assert np.array_equal(B.to_numpy(y), B.to_numpy(y1)) and np.array_equal(B.to_numpy(y), B.to_numpy(y0))
    z = device_z(B, D, N, SEED, off, col)
    assert rel(z, O.philox_normals(SEED, off, D, N, column_offset=col)) <= 1e-5
    y64, q64 = R.forward(ol, flags, z, mu, sigma, L)
    _, q32 = R.forward(ol, flags, z.astype(f32), mu, sigma, L, dtype=np.float32)
    assert rel(B.to_numpy(lq), q64) <= max(RTOL, (4 if chain in NETWORK else 2) * rel(q32, q64))
    if chain in ("planar8", "rqs_stacked", "radial_bn") and base_kind != "tril" and D in FUSED_D:
        assert launches == 1
    if chain in ("none", "planar_rqs_stacked", "permute_coupling", "rqs_stacked"):  # closed-form inverse: logpdf(td, y) agrees
        lp = B.logpdf(td, y)
        assert rel(B.to_numpy(lq), B.to_numpy(lp)) <= 1e-4


@pytest.mark.parametrize("chain,base_kind", [("planar8", "diag"), ("permute_coupling", "diag"), ("planar8", "tril")])
def test_ldy_wider_than_d(B, chain, base_kind):
    """Fused, two-pass and TRIL-base forward paths into a batch with ldy > D: the padding rows stay untouched."""
    import torch

    rng = np.random.default_rng(3)
    D, N = 64, 1000
    td, *_ = build(B, chain, D, rng, base_kind)
    from bijectors_jl_b200.interface import _desc_array, _stream
    from bijectors_jl_b200.transformed_distribution import _rsample_setup

    _, descs, _, base, _ = _rsample_setup(td, N, "test")
    arr, bd = _desc_array(descs), _desc_array([base])
    ld = 72
    buf = torch.full((N, ld), 7.0, device="cuda")
    lq = torch.empty(N, device="cuda")
    lib = B.lib()
    ws = torch.empty(lib.b2b_chain_sample_logq_workspace_bytes(arr, len(descs), bd, D, N), dtype=torch.uint8, device="cuda")
    rc = lib.b2b_chain_sample_logq_f32(arr, len(descs), bd, ctypes.c_uint64(SEED), ctypes.c_uint64(0), 0,
                                       buf.data_ptr(), lq.data_ptr(), D, N, ld, ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0
    y, lq2 = B.rand_logpdf(td, N, seed=SEED)
    assert np.array_equal(B.to_numpy(buf[:, :D].t()), B.to_numpy(y)) and np.array_equal(B.to_numpy(lq), B.to_numpy(lq2))
    assert float(buf[:, D:].min()) == 7.0 == float(buf[:, D:].max())


# ---- 4. gradients ------------------------------------------------------------------------------------------------------
def check_grads(B, td, ol, flags, mu, sigma, L, D, N, ybar, qbar, gate=2.0):
    import torch

    yb = None if ybar is None else B.from_numpy(ybar.astype(f32))
    qb = None if qbar is None else torch.from_numpy(qbar.astype(f32)).cuda()
    flow_g, base_g = B.rand_vjp(td, N, yb, qb, seed=SEED, offset=1, column_offset=5)
    z = device_z(B, D, N, SEED, 1, 5)
    base = td if isinstance(td, B.MvNormal) else td.dist
    x = B.to_numpy(base.rand(N, seed=SEED, offset=1, column_offset=5)).astype(np.float64)  # the x the chain saw
    g64, b64 = R.vjp(ol, flags, z, ybar, qbar, mu, sigma, L, x=x)
    g32, b32 = R.vjp(ol, flags, z.astype(f32), None if ybar is None else ybar.astype(f32),
                     None if qbar is None else qbar.astype(f32), mu, sigma, L, dtype=np.float32, x=x.astype(f32))

    def chk(dev, a64, a32, what):
        e, tol = rel(B.to_numpy(dev), a64), max(RTOL, gate * rel(a32, a64))
        if np.size(a64) == 1:  # a planar b̄ is one column sum: the gate of the planar VJP tests, 5e-5·max(|b̄|, √N)
            b64 = abs(float(np.ravel(a64)[0]))
            tol = max(tol, 5e-5 * max(b64, np.sqrt(N)) / max(b64, 1e-30))
        assert e <= tol, (what, e, tol)

    assert len(flow_g) == len(ol)
    for l, (gd, a, b) in enumerate(zip(flow_g, g64, g32)):
        assert set(gd) == set(a), (l, set(gd), set(a))
        for k in gd:
            chk(gd[k], np.reshape(a[k], gd[k].shape), np.reshape(b[k], gd[k].shape), (l, k))
    assert set(base_g) == set(b64)
    for k in base_g:
        chk(base_g[k], b64[k], b32[k], k)
    return flow_g, base_g


@pytest.mark.parametrize("which", ["ybar", "qbar", "both"])
@pytest.mark.parametrize("base_kind", ["diag", "tril"])
@pytest.mark.parametrize("chain,D", [("planar_rqs_stacked", 64), ("permute_coupling", 48), ("planar8", 128),
                                     ("inverse_planar", 32), ("rqs_stacked", 256), ("none", 40), ("radial_bn", 64),
                                     ("every_kind", 64), ("planar_rqs_mlprqs_perm_stacked", 64), ("deep_mlp", 48),
                                     ("permute_rqs", 256)])
def test_gradients(B, chain, D, base_kind, which):
    rng = np.random.default_rng(D + len(chain) * 3 + len(which))
    N = 2500
    td, ol, flags, mu, sigma, L = build(B, chain, D, rng, base_kind)
    ybar = rng.standard_normal((D, N)) if which != "qbar" else None
    qbar = rng.standard_normal(N) if which != "ybar" else None
    check_grads(B, td, ol, flags, mu, sigma, L, D, N, ybar, qbar, gate=4.0 if chain in NETWORK else 2.0)


# ---- 5. sharding, determinism, graph capture ---------------------------------------------------------------------------
@pytest.mark.parametrize("base_kind", ["diag", "tril"])
def test_shards_and_determinism(B, base_kind):
    import torch

    rng = np.random.default_rng(11)
    D, N, n0 = 64, 5000, 1937
    td, *_ = build(B, "planar_rqs_stacked", D, rng, base_kind)
    y, lq = B.rand_logpdf(td, N, seed=SEED, offset=2)
    ya, qa = B.rand_logpdf(td, n0, seed=SEED, offset=2)
    yb, qb = B.rand_logpdf(td, N - n0, seed=SEED, offset=2, column_offset=n0)
    assert np.array_equal(B.to_numpy(y), np.concatenate([B.to_numpy(ya), B.to_numpy(yb)], axis=1))
    assert np.array_equal(B.to_numpy(lq), np.concatenate([B.to_numpy(qa), B.to_numpy(qb)]))
    ybar = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    qbar = torch.from_numpy(rng.standard_normal(N).astype(f32)).cuda()
    f1, b1 = B.rand_vjp(td, N, ybar, qbar, seed=SEED, offset=2)
    f2, b2 = B.rand_vjp(td, N, ybar, qbar, seed=SEED, offset=2)
    fa, ba = B.rand_vjp(td, n0, ybar[:, :n0], qbar[:n0].contiguous(), seed=SEED, offset=2)
    fb, bb = B.rand_vjp(td, N - n0, ybar[:, n0:], qbar[n0:].contiguous(), seed=SEED, offset=2, column_offset=n0)
    for g1, g2, ga, gb in zip(f1 + [b1], f2 + [b2], fa + [ba], fb + [bb]):
        for k in g1:
            assert torch.equal(g1[k], g2[k]), k
            assert rel(B.to_numpy(ga[k] + gb[k]), B.to_numpy(g1[k])) <= 1e-5, k


def test_graph_capture(B):
    import torch

    from bijectors_jl_b200.interface import _desc_array, _stream
    from bijectors_jl_b200.transformed_distribution import _rsample_setup

    rng = np.random.default_rng(12)
    D, N = 64, 4096
    td, *_ = build(B, "permute_coupling", D, rng, "diag")
    _, descs, _, base, _ = _rsample_setup(td, N, "test")
    arr, bd = _desc_array(descs), _desc_array([base])
    lib, L = B.lib(), len(descs)
    y_ref, lq_ref = B.rand_logpdf(td, N, seed=SEED)
    ws1 = torch.empty(lib.b2b_chain_sample_logq_workspace_bytes(arr, L, bd, D, N), dtype=torch.uint8, device="cuda")
    wsv = torch.empty(lib.b2b_chain_sample_vjp_workspace_bytes(arr, L, bd, D, N), dtype=torch.uint8, device="cuda")
    y = B.colmajor_empty(D, N)
    lq = torch.empty(N, device="cuda")
    mubar, sbar = torch.empty(D, device="cuda"), torch.empty(D, device="cuda")
    bars = (ctypes.c_void_p * (4 * (L + 1)))()
    bars[4 * L], bars[4 * L + 1] = mubar.data_ptr(), sbar.data_ptr()
    lqbar = torch.ones(N, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        st = torch.cuda.current_stream().cuda_stream
        rc1 = lib.b2b_chain_sample_logq_f32(arr, L, bd, ctypes.c_uint64(SEED), ctypes.c_uint64(0), 0, y.data_ptr(),
                                            lq.data_ptr(), D, N, D, ws1.data_ptr(), ws1.numel(), st)
        rc2 = lib.b2b_chain_sample_vjp_f32(arr, L, bd, ctypes.c_uint64(SEED), ctypes.c_uint64(0), 0, None, D,
                                           lqbar.data_ptr(), bars, D, N, wsv.data_ptr(), wsv.numel(), st)
    assert rc1 == 0 and rc2 == 0
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, y_ref) and torch.equal(lq, lq_ref)
    _, bg = B.rand_vjp(td, N, None, lqbar, seed=SEED)
    assert torch.equal(mubar, bg["μ"]) and torch.equal(sbar, bg["σ"])


# ---- 6. refusals -------------------------------------------------------------------------------------------------------
def test_refusals(B):
    import torch

    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200.interface import _desc_array, _stream
    from bijectors_jl_b200.transformed_distribution import _rsample_setup

    lib = B.lib()
    rng = np.random.default_rng(13)
    y = B.colmajor_empty(300, 64)
    lq = torch.empty(64, device="cuda")

    def call(td, D, bars=None):
        _, descs, _, base, _ = _rsample_setup(td, 64, "test")
        arr = _desc_array(descs) if descs else None
        bd = _desc_array([base])
        L = len(descs)
        rc1 = lib.b2b_chain_sample_logq_f32(arr, L, bd, ctypes.c_uint64(1), ctypes.c_uint64(0), 0, y.data_ptr(),
                                            lq.data_ptr(), D, 64, 300, None, 0, _stream())
        n1 = lib.b2b_last_launch_count()
        rc2 = lib.b2b_chain_sample_vjp_f32(arr, L, bd, ctypes.c_uint64(1), ctypes.c_uint64(0), 0, None, D, None, bars,
                                           D, 64, None, 0, _stream())
        n2 = lib.b2b_last_launch_count()
        return (rc1, n1, lib.b2b_chain_sample_logq_workspace_bytes(arr, L, bd, D, 64), rc2, n2,
                lib.b2b_chain_sample_vjp_workspace_bytes(arr, L, bd, D, 64))

    # a TRIL base with D = 257
    base = B.MvNormal(257, scale_tril=np.eye(257, dtype=f32))
    assert call(base, 257) == (_lib.B2B_EUNSUPPORTED, 0, 0, _lib.B2B_EUNSUPPORTED, 0, 0)
    # an unsupported chain: a planar layer at D = 300 has no reverse-mode kernel
    td = B.transformed(B.MvNormal(300), planar(B, 300, rng)[0])
    rc1, n1, w1, rc2, n2, w2 = call(td, 300)
    assert rc1 == rc2 == _lib.B2B_EUNSUPPORTED and n1 == n2 == 0 and w1 == w2 == 0
    # a μ̄ request for a base without μ
    td = B.transformed(B.MvNormal(64), planar(B, 64, rng)[0])
    bars = (ctypes.c_void_p * 8)()
    bars[4] = lq.data_ptr()
    assert call(td, 64, bars)[3] == _lib.B2B_EINVAL


# ---- 7. autograd ---------------------------------------------------------------------------------------------------------
def test_flow_rsample_matches_rand_vjp(B):
    import torch

    rng = np.random.default_rng(21)
    D, N = 32, 2000
    td, ol, flags, mu, sigma, L = build(B, "inverse_planar", D, rng, "tril")
    flow = B.autograd.Flow(td.transform, td.dist)
    y, lq = flow.rsample(N, seed=SEED)
    ybar = torch.from_numpy(rng.standard_normal((D, N)).astype(f32)).cuda()
    loss = (y * ybar).sum() + lq.sum()
    loss.backward()
    fg, bg = B.rand_vjp(td, N, B.from_numpy(B.to_numpy(ybar)), torch.ones(N, device="cuda"), seed=SEED)
    expect = {}
    for g, leaf in zip(fg, B.flatten(td.transform)):
        from bijectors_jl_b200.autograd import _trainable_tensors

        for t, k in zip(_trainable_tensors(leaf), g):
            expect.setdefault(t.data_ptr(), 0)
            expect[t.data_ptr()] = expect[t.data_ptr()] + g[k].reshape(t.shape)
    expect[td.dist.mu.data_ptr()] = bg["μ"]
    expect[td.dist._tril.data_ptr()] = bg["L"].t()
    for p in flow.params:
        assert torch.allclose(p.grad, expect[p.data_ptr()], rtol=1e-6, atol=1e-6)


def test_elbo_fit(B):
    """Fit q = planar flow over a trainable diagonal base to a Gaussian target p by maximising the ELBO."""
    import torch

    rng = np.random.default_rng(31)
    D, N = 32, 8192
    tmu = (rng.standard_normal(D) * 1.0).astype(f32)
    tsig = rng.uniform(0.5, 2.0, D).astype(f32)
    layers = [planar(B, D, rng, 0.1)[0] for _ in range(4)]
    base = B.MvNormal(D, mu=np.zeros(D, f32), sigma=np.ones(D, f32))
    flow = B.autograd.Flow(B.Composed(*layers), base)
    tm, ts = torch.from_numpy(tmu).cuda(), torch.from_numpy(tsig).cuda()

    def kl_estimate(seed):
        y, lq = flow.rsample(N, seed=seed)
        lp = (-0.5 * (((y - tm[:, None]) / ts[:, None]) ** 2).sum(0) - torch.log(ts).sum() - 0.5 * D * np.log(2 * np.pi))
        return (lq - lp).mean()

    # the first gradient against the float64 reference
    kl = kl_estimate(77)
    kl.backward()
    td = B.transformed(base, flow.transform)
    y = B.to_numpy(B.rand(td, N, seed=77)).astype(np.float64)
    ybar = (y - tmu[:, None].astype(np.float64)) / tsig[:, None].astype(np.float64) ** 2 / N  # ∂(−log p / N)/∂y
    z = device_z(B, D, N, 77, 0, 0)
    ol = [O.Layer("planar", dict(w=B.to_numpy(l.w), u=B.to_numpy(l.u), b=B.to_numpy(l.b))) for l in layers]
    g64, b64 = R.vjp(ol, [False] * 4, z, ybar, np.full(N, 1.0 / N), B.to_numpy(base.mu), B.to_numpy(base.sigma))
    g32, b32 = R.vjp(ol, [False] * 4, z.astype(f32), ybar.astype(f32), np.full(N, 1.0 / N, f32), B.to_numpy(base.mu),
                     B.to_numpy(base.sigma), dtype=np.float32)
    grad = {p.data_ptr(): p.grad for p in flow.params}
    for t, a64, a32 in [(base.mu, b64["μ"], b32["μ"]), (base.sigma, b64["σ"], b32["σ"]),
                        (layers[0].w, g64[0]["w"], g32[0]["w"]), (layers[3].u, g64[3]["u"], g32[3]["u"])]:
        # the target's log-density is formed in float32 torch arithmetic: 1e-4 covers its rounding in ȳ
        assert rel(B.to_numpy(grad[t.data_ptr()]), a64) <= max(1e-4, 2 * rel(a32, a64))
    opt = torch.optim.Adam(flow.parameters(), lr=2e-2)
    opt.zero_grad()
    with torch.no_grad():
        k0 = float(np.mean([float(kl_estimate(1000 + i)) for i in range(4)]))
    for step in range(300):
        opt.zero_grad()
        kl_estimate(step).backward()
        opt.step()
    with torch.no_grad():
        k1 = float(np.mean([float(kl_estimate(2000 + i)) for i in range(4)]))
    assert k1 < 0.5 * k0, (k0, k1)


def test_float64_and_bad_base_raise(B):
    import torch

    base = B.MvNormal(8, mu=np.zeros(8), sigma=np.ones(8), dtype=torch.float64)
    with pytest.raises(TypeError):
        B.rand_logpdf(base, 10, seed=1)
    with pytest.raises(TypeError):
        B.rand_vjp(base, 10, seed=1)
