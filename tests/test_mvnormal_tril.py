"""GPU tests of the full-covariance MvNormal base (B2B_MVNORMAL_TRIL): logpdf, reverse mode and sampling against the float64
reference of tests/mvnormal_tril_oracle.py.  Gates are tied to the reference's own float32 error on the same input, as in
test_chain_vjp.py: max(1e-5, 2 × ‖oracle32 − oracle64‖ / ‖oracle64‖), norm-wise."""
import ctypes
import math

import numpy as np
import pytest

import chain_vjp_oracle as V
import mvnormal_tril_oracle as T
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(dev, a64, a32, what=""):
    tol = max(RTOL, 2.0 * rel(a32, a64))
    e = rel(dev, a64)
    assert e <= tol, (what, e, tol)


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def case(rng, D, N, with_mu=True):
    L = T.random_tril(rng, D).astype(f32)
    mu = (rng.standard_normal(D) * 0.3).astype(f32) if with_mu else None
    x = (rng.standard_normal((D, N))).astype(f32)
    return L, mu, x


def base(B, L, mu):
    return B.MvNormal(L.shape[0], mu=mu, scale_tril=L)


def tril_desc(B, L_dev_colmajor, mu_dev=None):
    d = B._lib.LayerDesc()
    d.kind = B._lib.MVNORMAL_TRIL
    d.p0 = mu_dev.data_ptr() if mu_dev is not None else None
    d.p1 = L_dev_colmajor.data_ptr() if L_dev_colmajor is not None else None
    return d


def stream():
    import torch

    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- logpdf parity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 5, 1000, 65539])
@pytest.mark.parametrize("D", [1, 3, 32, 64, 100, 128, 255, 256])
def test_logpdf_parity(B, D, N):
    rng = np.random.default_rng(D * 7 + N)
    L, mu, x = case(rng, D, N)
    lp = B.to_numpy(B.logpdf(base(B, L, mu), B.from_numpy(x)))
    gate(lp, T.logpdf(L, mu, x), T.logpdf(L, mu, x, np.float32), (D, N))


def test_logpdf_ill_conditioned_factor(B):
    rng = np.random.default_rng(3)
    D, N = 64, 2000
    L = T.random_tril(rng, D, cond=1e3).astype(f32)
    x = (L.astype(np.float64) @ rng.standard_normal((D, N))).astype(f32)
    lp = B.to_numpy(B.logpdf(base(B, L, None), B.from_numpy(x)))
    gate(lp, T.logpdf(L, None, x), T.logpdf(L, None, x, np.float32))


def planar_pair(B, D, rng, scale):
    w, u = (rng.standard_normal(D) * scale).astype(f32), (rng.standard_normal(D) * scale).astype(f32)
    b = rng.standard_normal(1).astype(f32)
    return B.PlanarLayer(w, u, b), O.Layer("planar", dict(w=w, u=u, b=b))


def chain(B, kind, D, rng):
    """(flow, oracle layers of inverse(flow) in application order, inverse flags)."""
    if kind == "planar":
        pairs = [planar_pair(B, D, rng, 0.1) for _ in range(4)]
        flow = B.Composed(*[p for p, _ in pairs])
        return flow, [o for _, o in pairs][::-1], [True] * 4
    if kind == "radial":
        a, be = rng.standard_normal(1).astype(f32), rng.standard_normal(1).astype(f32)
        z0 = (rng.standard_normal(D) * 0.3).astype(f32)
        return B.RadialLayer(a, be, z0), [O.Layer("radial", dict(alpha_raw=a, beta=be, z0=z0))], [True]
    if kind == "coupling":
        n1 = D // 2
        W = (rng.standard_normal((2 * n1, D - n1)) * 0.01).astype(f32)
        c = (rng.standard_normal(2 * n1) * 0.1).astype(f32)
        idx1, idx2 = list(range(1, n1 + 1)), list(range(n1 + 1, D + 1))
        cp = B.Coupling(B.AffineConditioner(W, c), B.PartitionMask(D, idx1, idx2))
        return cp, [O.Layer("coupling_affine", dict(idx1=np.asarray(idx1), idx2=np.asarray(idx2), W=W, c=c))], [True]
    if kind == "stacked_permute":
        half = D // 2
        st = B.Stacked([B.Shift(0.7), B.Scale(-1.7)], [(1, half), (half + 1, D)])
        ost = O.Layer("stacked", dict(ops=[(O.EW.SHIFT, f32(0.7)), (O.EW.SCALE, f32(-1.7))], ranges=[(1, half), (half + 1, D)]))
        perm = (rng.permutation(D) + 1).tolist()
        flow = B.Composed(st, B.Permute(perm))
        return flow, [O.Layer("permute", dict(A=O.permute_matrix_from_indices(perm))), ost], [True, True]
    raise ValueError(kind)


KINDS = ["planar", "radial", "coupling", "stacked_permute"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D,N", [(64, 3001), (100, 517)])
def test_logpdf_after_inverse_chain(B, kind, D, N):
    rng = np.random.default_rng(D + len(kind))
    L, mu, y = case(rng, D, N)
    flow, ol, flags = chain(B, kind, D, rng)
    td = B.transformed(base(B, L, mu), flow)
    lp = B.to_numpy(B.logpdf(td, B.from_numpy(y)))
    gate(lp, V.chain_logjac(ol, flags, y, mu, scale_tril=L)[1],
         V.chain_logjac(ol, flags, y.astype(f32), mu, dtype=np.float32, scale_tril=L)[1], kind)
    s, lp2 = B.logpdf_sum(td, B.from_numpy(y))
    assert abs(float(s) - float(lp2.double().sum())) <= 1e-9 * max(1.0, abs(float(s)))


def test_layouts_and_batch_sum(B):
    """Padded ld, a misaligned batch, y given or NULL, and sum_out bit-identical across repeats (raw C ABI)."""
    import torch

    lib = B.lib()
    rng = np.random.default_rng(17)
    D, N = 100, 4099
    L, mu, x = case(rng, D, N)
    ref = T.logpdf(L, mu, x)
    ref32 = T.logpdf(L, mu, x, np.float32)
    Ld = torch.from_numpy(np.ascontiguousarray(L.T)).cuda()  # column-major L
    mud = torch.from_numpy(mu).cuda()
    arr = (B._lib.LayerDesc * 1)(tril_desc(B, Ld, mud))
    for ld, off in [(D, 0), (D + 7, 0), (D + 3, 1)]:
        buf = torch.full((ld * N + off + 8,), float("nan"), device="cuda")
        xv = buf[off:off + ld * N].view(N, ld)
        xv[:, :D] = torch.from_numpy(x.T.copy()).cuda()
        for want_y in (False, True):
            y = torch.full((N, ld), float("nan"), device="cuda") if want_y else None
            lj = torch.empty(N, device="cuda")
            s = torch.empty((), dtype=torch.float64, device="cuda")
            ws_b = lib.b2b_chain_workspace_bytes(arr, 1, D, N, int(want_y), 1)
            ws = torch.empty(max(ws_b, 1), dtype=torch.uint8, device="cuda")
            sums = []
            for _ in range(2):
                rc = lib.b2b_chain_run_f32(arr, 1, xv.data_ptr(), y.data_ptr() if want_y else None, lj.data_ptr(),
                                           s.data_ptr(), D, N, ld, ld, 0, ws.data_ptr(), ws_b, stream())
                assert rc == 0
                torch.cuda.synchronize()
                sums.append(float(s))
            gate(lj.cpu().numpy(), ref, ref32, (ld, off, want_y))
            assert sums[0] == sums[1]
            assert abs(sums[0] - float(lj.double().sum())) <= 1e-9 * abs(sums[0])
            if want_y:
                assert torch.equal(y[:, :D], xv[:, :D])


def test_consistency_with_diagonal_and_standard_base(B):
    rng = np.random.default_rng(23)
    D, N = 128, 3000
    sig = rng.uniform(0.5, 2.0, D).astype(f32)
    mu = rng.standard_normal(D).astype(f32)
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    a = B.to_numpy(B.logpdf(B.MvNormal(D, mu=mu, scale_tril=np.diag(sig)), x))
    b = B.to_numpy(B.logpdf(B.MvNormal(D, mu=mu, sigma=sig), x))
    xs = B.to_numpy(x)
    gate(a, O.mvnormal_diag_logpdf(mu.astype(np.float64), sig.astype(np.float64), xs.astype(np.float64)),
         O.mvnormal_diag_logpdf(mu, sig, xs), "diag")
    assert rel(a, b) <= 2e-6
    c = B.to_numpy(B.logpdf(B.MvNormal(D, scale_tril=np.eye(D, dtype=f32)), x))
    d = B.to_numpy(B.logpdf(B.MvNormal(D), x))
    assert rel(c, d) <= 2e-6
    e = B.to_numpy(B.logpdf(B.MvNormal(D, mu=mu, cov=np.diag(sig.astype(np.float64) ** 2)), x))
    assert rel(e, b) <= 2e-6


# ---- reverse mode ---------------------------------------------------------------------------------------------------------
def check_vjp(B, td, ol, flags, y, lb, L, mu):
    import torch

    yb, flow_g, base_g = B.logpdf_vjp(td, B.from_numpy(y), torch.from_numpy(lb.astype(f32)).cuda())
    o64 = V.chain_vjp(ol, flags, y, None, lb, mu, scale_tril=L)
    o32 = V.chain_vjp(ol, flags, y.astype(f32), None, lb, mu, dtype=np.float32, scale_tril=L)
    gate(B.to_numpy(yb), o64[0], o32[0], "x̄")
    assert set(base_g) == set(o64[2])
    for k in base_g:
        gate(base_g[k].cpu().numpy(), o64[2][k], o32[2][k], k)
    Lb = base_g["L"].cpu().numpy()
    assert np.all(np.triu(Lb, 1) == 0.0)
    dev = flow_g[::-1]
    for l, (gd, g64, g32) in enumerate(zip(dev, o64[1], o32[1])):
        for k in gd:
            gate(gd[k].cpu().numpy().reshape(-1), np.reshape(g64[k], -1), np.reshape(g32[k], -1), (l, k))


@pytest.mark.parametrize("D,N", [(1, 7), (3, 1000), (32, 513), (100, 4097), (256, 1000)])
def test_vjp_terminal_alone(B, D, N):
    rng = np.random.default_rng(D * 3 + N)
    L, mu, y = case(rng, D, N)
    lb = rng.standard_normal(N)
    import torch

    d = B.MvNormal(D, mu=mu, scale_tril=L)
    descs = [d._terminal_desc()]
    from bijectors_jl_b200.interface import _chain_vjp_raw

    xb, bars = _chain_vjp_raw(descs, B.from_numpy(y), None, torch.from_numpy(lb.astype(f32)).cuda(), [(0, 0), (0, 1)])
    g64, m64, L64 = T.logpdf_vjp(L, mu, y, lb)
    g32, m32, L32 = T.logpdf_vjp(L, mu, y, lb, np.float32)
    gate(B.to_numpy(xb), g64, g32, "x̄")
    gate(bars[(0, 0)].cpu().numpy(), m64, m32, "μ̄")
    Lb = bars[(0, 1)].t().cpu().numpy()
    gate(Lb, L64, L32, "L̄")
    assert np.all(np.triu(Lb, 1) == 0.0)


@pytest.mark.parametrize("kind", KINDS)
def test_vjp_through_chains(B, kind):
    rng = np.random.default_rng(31 + len(kind))
    D, N = 64, 2049
    L, mu, y = case(rng, D, N)
    flow, ol, flags = chain(B, kind, D, rng)
    check_vjp(B, B.transformed(base(B, L, mu), flow), ol, flags, y, rng.standard_normal(N), L, mu)


def test_vjp_without_mu_and_status_codes(B):
    import torch

    lib = B.lib()
    rng = np.random.default_rng(41)
    D, N = 16, 100
    L, _, x = case(rng, D, N, with_mu=False)
    Ld = torch.from_numpy(np.ascontiguousarray(L.T)).cuda()
    arr = (B._lib.LayerDesc * 1)(tril_desc(B, Ld, None))
    xd = B.from_numpy(x)
    xb = torch.empty_like(xd)
    ws_b = lib.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
    assert ws_b > 0
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    out = torch.empty(D * D, device="cuda")
    for slot, want in [(0, B._lib.B2B_EINVAL), (2, B._lib.B2B_EUNSUPPORTED), (3, B._lib.B2B_EUNSUPPORTED)]:
        ptrs = (ctypes.c_void_p * 4)()
        ptrs[slot] = out.data_ptr()
        rc = lib.b2b_chain_vjp_f32(arr, 1, xd.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(ptrs, ctypes.c_void_p), D,
                                   N, D, D, D, ws.data_ptr(), ws_b, stream())
        assert rc == want, (slot, rc)
    ptrs = (ctypes.c_void_p * 4)()
    ptrs[1] = out.data_ptr()
    lb = torch.from_numpy(rng.standard_normal(N).astype(f32)).cuda()
    rc = lib.b2b_chain_vjp_f32(arr, 1, xd.data_ptr(), None, lb.data_ptr(), xb.data_ptr(), ctypes.cast(ptrs, ctypes.c_void_p),
                               D, N, D, D, D, ws.data_ptr(), ws_b, stream())
    assert rc == 0
    _, _, L64 = T.logpdf_vjp(L, None, x, lb.cpu().numpy().astype(np.float64))
    _, _, L32 = T.logpdf_vjp(L, None, x, lb.cpu().numpy(), np.float32)
    gate(out.view(D, D).t().cpu().numpy(), L64, L32)


def test_flow_routes_mu_and_L(B):
    import torch

    rng = np.random.default_rng(43)
    D, N = 32, 1500
    L, mu, y = case(rng, D, N)
    flow, ol, flags = chain(B, "planar", D, rng)
    bse = base(B, L, mu)
    F = B.autograd.Flow(flow, base=bse)
    ptrs = {p.data_ptr(): p for p in F.params}
    assert bse.mu.data_ptr() in ptrs and bse._tril.data_ptr() in ptrs
    F.nll(B.from_numpy(y)).backward()
    lb = np.full(N, -1.0)
    o64 = V.chain_vjp(ol, flags, y, None, lb, mu, scale_tril=L)
    o32 = V.chain_vjp(ol, flags, y.astype(f32), None, lb, mu, dtype=np.float32, scale_tril=L)
    gate(ptrs[bse.mu.data_ptr()].grad.cpu().numpy(), o64[2]["μ"], o32[2]["μ"], "μ")
    gate(ptrs[bse._tril.data_ptr()].grad.t().cpu().numpy(), o64[2]["L"], o32[2]["L"], "L")


# ---- sampling -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 3, 64, 100, 256])
def test_rand_is_unwhitened_philox_stream(B, D):
    rng = np.random.default_rng(D + 5)
    N = 3001
    L, mu, _ = case(rng, D, N)
    d = base(B, L, mu)
    y = B.to_numpy(d.rand(N, seed=1234, offset=3))
    z = O.philox_normals(1234, 3, D, N)
    ref = T.sample(L, mu, z)
    ref32 = (mu[:, None] + (L @ z.astype(f32))).astype(f32)
    gate(y, ref, ref32, D)
    y2 = B.to_numpy(d.rand(N, seed=1234, offset=3))
    assert np.array_equal(y, y2)
    tail = B.to_numpy(d.rand(1000, seed=1234, offset=3, column_offset=2001))
    assert np.array_equal(tail, y[:, 2001:])


def test_rand_through_flow_equals_run_chain(B):
    rng = np.random.default_rng(51)
    D, N = 64, 4097
    L, mu, _ = case(rng, D, N)
    flow, _, _ = chain(B, "planar", D, rng)
    td = B.transformed(base(B, L, mu), flow)
    y, lj = B.rand(td, N, seed=9, with_logjac=True)
    x = B.rand(td.dist, N, seed=9)
    y2, lj2 = B.run_chain(flow, x)
    assert B.to_numpy(y).tobytes() == B.to_numpy(y2).tobytes()
    assert B.to_numpy(lj).tobytes() == B.to_numpy(lj2).tobytes()


def test_rand_covariance(B):
    import torch

    rng = np.random.default_rng(61)
    D, N = 8, 1 << 20
    L = T.random_tril(rng, D).astype(f32)
    mu = rng.standard_normal(D).astype(f32)
    y = B.MvNormal(D, mu=mu, scale_tril=L).rand(N, seed=77).double()
    m = y.mean(dim=1).cpu().numpy()
    C = torch.cov(y).cpu().numpy()
    S = L.astype(np.float64) @ L.T.astype(np.float64)
    sd = np.sqrt(np.diag(S))
    # sampling error of an entry of the empirical covariance: sqrt((S_ij² + S_ii S_jj) / N); 6 of those
    tol = 6.0 * np.sqrt((S * S + np.outer(np.diag(S), np.diag(S))) / N)
    assert np.all(np.abs(C - S) <= tol)
    assert np.all(np.abs(m - mu) <= 6.0 * sd / math.sqrt(N))


# ---- limits and status codes ----------------------------------------------------------------------------------------------
def test_d257_is_refused_before_launching(B):
    import torch

    lib = B.lib()
    D, N = 257, 64
    L = torch.eye(D, device="cuda")
    arr = (B._lib.LayerDesc * 1)(tril_desc(B, L))
    x = torch.zeros((N, D), device="cuda")
    lj = torch.full((N,), float("nan"), device="cuda")
    y = torch.full((N, D), float("nan"), device="cuda")
    assert lib.b2b_chain_workspace_bytes(arr, 1, D, N, 1, 1) == 0
    assert lib.b2b_workspace_bytes(arr, D, N) == 0
    assert lib.b2b_chain_vjp_workspace_bytes(arr, 1, D, N) == 0
    rc = lib.b2b_chain_run_f32(arr, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream())
    assert rc == B._lib.B2B_EUNSUPPORTED and lib.b2b_last_launch_count() == 0
    xb = torch.full((N, D), float("nan"), device="cuda")
    rc = lib.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, None, 0, stream())
    assert rc == B._lib.B2B_EUNSUPPORTED and lib.b2b_last_launch_count() == 0
    rc = lib.b2b_chain_sample_tril_f32(None, 0, None, L.data_ptr(), 1, 0, 0, y.data_ptr(), lj.data_ptr(), D, N, D, None, 0,
                                       stream())
    assert rc == B._lib.B2B_EUNSUPPORTED and lib.b2b_last_launch_count() == 0
    torch.cuda.synchronize()
    assert torch.isnan(lj).all() and torch.isnan(y).all() and torch.isnan(xb).all()


def test_einval_cases(B):
    import torch

    lib = B.lib()
    D, N = 8, 16
    L = torch.eye(D, device="cuda")
    x = torch.zeros((N, D), device="cuda")
    lj = torch.empty(N, device="cuda")
    t = tril_desc(B, L)
    p = B._lib.LayerDesc()
    p.kind = B._lib.PERMUTE
    perm = torch.arange(D, dtype=torch.int32, device="cuda")
    p.i0 = perm.data_ptr()
    inv = tril_desc(B, L)
    inv.inverse = 1
    nul = tril_desc(B, None)
    bad = tril_desc(B, L)
    bad.kind = 10
    for descs in ([t, p], [inv], [nul], [bad]):
        arr = (B._lib.LayerDesc * len(descs))(*descs)
        rc = lib.b2b_chain_run_f32(arr, len(descs), x.data_ptr(), None, lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream())
        assert rc == B._lib.B2B_EINVAL
    rc = lib.b2b_chain_sample_tril_f32(None, 0, None, None, 1, 0, 0, x.data_ptr(), None, D, N, D, None, 0, stream())
    assert rc == B._lib.B2B_EINVAL


def test_host_buffer_path_is_bit_identical(B):
    import torch

    rng = np.random.default_rng(71)
    D, N = 64, 20000
    L, mu, y = case(rng, D, N)
    flow, _, _ = chain(B, "planar", D, rng)
    td = B.transformed(base(B, L, mu), flow)
    dev = B.to_numpy(B.logpdf(td, B.from_numpy(y)))
    host = B.logpdf(td, B.from_numpy(y).cpu())
    assert not host.is_cuda
    assert host.numpy().tobytes() == dev.tobytes()


def test_deterministic_and_graph_capture(B):
    import torch

    rng = np.random.default_rng(81)
    D, N = 128, 20000
    L, mu, y = case(rng, D, N)
    flow, _, _ = chain(B, "planar", D, rng)
    td = B.transformed(base(B, L, mu), flow)
    yd = B.from_numpy(y)
    lb = torch.randn(N, device="cuda")
    a = (B.logpdf(td, yd), *B.logpdf_vjp(td, yd, lb))
    b = (B.logpdf(td, yd), *B.logpdf_vjp(td, yd, lb))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(a[3][k], b[3][k]) for k in a[3])
    out = {}
    g = B.GraphedCalls(lambda: out.__setitem__("r", (B.logpdf(td, yd), *B.logpdf_vjp(td, yd, lb))))
    c = out["r"]
    c[0].fill_(float("nan"))
    c[1].fill_(float("nan"))
    c[3]["L"].fill_(float("nan"))
    g()
    torch.cuda.synchronize()
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1]) and all(torch.equal(a[3][k], c[3][k]) for k in a[3])


def test_training_fits_covariance(B):
    import torch

    rng = np.random.default_rng(91)
    D, N = 8, 8192
    A = T.random_tril(rng, D) * 1.5
    S = A @ A.T
    data = B.from_numpy((A @ rng.standard_normal((D, N))).astype(f32))
    flow = B.Composed(*[B.PlanarLayer((rng.standard_normal(D) * 0.01).astype(f32), (rng.standard_normal(D) * 0.01).astype(f32),
                                      np.zeros(1, f32)) for _ in range(4)])
    bse = B.MvNormal(D, mu=np.zeros(D, f32), scale_tril=np.eye(D, dtype=f32))
    F = B.autograd.Flow(flow, base=bse)
    opt = torch.optim.Adam(F.params, lr=2e-2)
    losses = []
    start = rel(np.eye(D), S)
    for _ in range(300):
        opt.zero_grad()
        loss = F.nll(data) / N
        loss.backward()
        opt.step()
        with torch.no_grad():  # keep L lower triangular with a positive diagonal (what a Cholesky factor is)
            Lt = bse._tril.t()
            Lt.copy_(torch.tril(Lt))
            Lt.diagonal().clamp_(min=1e-3)
        losses.append(float(loss))
    assert losses[-1] < losses[0] - 1.0
    Lf = bse.scale_tril.detach().cpu().numpy().astype(np.float64)
    assert rel(Lf @ Lf.T, S) < 0.5 * start, (rel(Lf @ Lf.T, S), start)


def test_batch_sum_without_logjac_after_layers(B):
    """A TRIL-terminated chain with layers before it takes sum_out with logjac = NULL, as MVNORMAL_DIAG does: the layers'
    log-Jacobians go through the workspace."""
    import torch

    from bijectors_jl_b200.interface import _desc_array

    lib = B.lib()
    rng = np.random.default_rng(19)
    D, N = 64, 5003
    L, mu, y = case(rng, D, N)
    flow, ol, flags = chain(B, "planar", D, rng)
    bse = base(B, L, mu)
    descs = list(B.inverse(flow)._descs(False, D)) + [bse._terminal_desc()]
    arr = _desc_array(descs)
    yd = B.from_numpy(y)
    ws_b = lib.b2b_chain_workspace_bytes(arr, len(descs), D, N, 0, 1)
    assert ws_b >= lib.b2b_chain_workspace_bytes(arr, len(descs), D, N, 0, 0) + 4 * N
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    s = torch.empty((), dtype=torch.float64, device="cuda")
    rc = lib.b2b_chain_run_f32(arr, len(descs), yd.data_ptr(), None, None, s.data_ptr(), D, N, D, D, 0, ws.data_ptr(), ws_b,
                               stream())
    assert rc == 0
    ref = float(V.chain_logjac(ol, flags, y, mu, scale_tril=L)[1].sum())
    s_lj, _ = B.logpdf_sum(B.transformed(bse, flow), yd)
    assert float(s) == float(s_lj)
    assert abs(float(s) - ref) <= 1e-5 * abs(ref)
    rc = lib.b2b_chain_run_f32(arr, len(descs), yd.data_ptr(), None, None, s.data_ptr(), D, N, D, D, 0, ws.data_ptr(),
                               ws_b - 4 * N - 1024, stream())
    assert rc == B._lib.B2B_EWORKSPACE


# ---- Float64 --------------------------------------------------------------------------------------------------------------
TOL64 = 1e-10


def planar_pair64(B, D, rng, scale):
    import torch

    w, u, b = rng.standard_normal(D) * scale, rng.standard_normal(D) * scale, rng.standard_normal(1)
    return B.PlanarLayer(w, u, b, dtype=torch.float64), O.Layer("planar", dict(w=w, u=u, b=b))


@pytest.mark.parametrize("D", [3, 33, 128, 1000, 2048])
def test_float64_run_and_vjp(B, D):
    import torch

    rng = np.random.default_rng(D + 1000)
    N = 9
    L = T.random_tril(rng, D)
    mu = rng.standard_normal(D) * 0.3
    y = rng.standard_normal((D, N))
    pairs = [planar_pair64(B, D, rng, 0.1) for _ in range(2)]
    flow = B.Composed(*[p for p, _ in pairs])
    ol, flags = [o for _, o in pairs][::-1], [True, True]
    td = B.transformed(B.MvNormal(D, mu=mu, scale_tril=L, dtype=torch.float64), flow)
    yd = B.from_numpy(y, dtype=np.float64)
    lp = B.logpdf(td, yd)
    assert lp.dtype == torch.float64
    assert rel(lp.cpu().numpy(), V.chain_logjac(ol, flags, y, mu, scale_tril=L)[1]) <= TOL64
    lb = rng.standard_normal(N)
    yb, flow_g, base_g = B.logpdf_vjp(td, yd, torch.from_numpy(lb).cuda())
    o = V.chain_vjp(ol, flags, y, None, lb, mu, scale_tril=L)
    assert rel(B.to_numpy(yb), o[0]) <= TOL64
    assert rel(base_g["μ"].cpu().numpy(), o[2]["μ"]) <= TOL64
    Lb = base_g["L"].cpu().numpy()
    assert rel(Lb, o[2]["L"]) <= TOL64 and np.all(np.triu(Lb, 1) == 0.0)
    for gd, g64 in zip(flow_g[::-1], o[1]):
        for k in gd:
            dev, ref = gd[k].cpu().numpy().reshape(-1), np.reshape(g64[k], -1)
            if ref.size == 1:  # planar b̄: one column sum, held like the Float64 chain tests hold it
                assert abs(dev[0] - ref[0]) <= TOL64 * max(abs(ref[0]), 1e-2 * math.sqrt(N)), k
            else:
                assert rel(dev, ref) <= TOL64, k


def test_gradcheck_flow_logpdf_f64(B):
    import torch

    rng = np.random.default_rng(77)
    D, N = 4, 3
    pairs = [planar_pair64(B, D, rng, 0.3) for _ in range(2)]
    bse = B.MvNormal(D, mu=rng.standard_normal(D) * 0.2, scale_tril=T.random_tril(rng, D), dtype=torch.float64)
    model = B.autograd.Flow(B.Composed(*[p for p, _ in pairs]), bse)
    ps = list(model.params)
    assert any(p.data_ptr() == bse._tril.data_ptr() for p in ps) and any(p.data_ptr() == bse.mu.data_ptr() for p in ps)
    y = B.from_numpy(rng.standard_normal((D, N)), dtype=np.float64).requires_grad_()
    assert torch.autograd.gradcheck(lambda y_, *p: model.logpdf(y_), (y, *ps), eps=1e-6, atol=1e-7, rtol=1e-5)


def test_float64_d2049_refused_and_status_codes(B):
    import torch

    lib = B.lib()
    D, N = 2049, 8
    Lm = torch.eye(D, dtype=torch.float64, device="cuda")
    d = B._lib.LayerDesc64()
    d.kind = B._lib.MVNORMAL_TRIL
    d.p1 = Lm.data_ptr()
    arr = (B._lib.LayerDesc64 * 1)(d)
    x = torch.zeros((N, D), dtype=torch.float64, device="cuda")
    lj = torch.full((N,), float("nan"), dtype=torch.float64, device="cuda")
    xb = torch.full((N, D), float("nan"), dtype=torch.float64, device="cuda")
    assert lib.b2b_chain_vjp_workspace_bytes_f64(arr, 1, D, N) == 0
    rc = lib.b2b_chain_run_f64(arr, 1, x.data_ptr(), None, lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream())
    assert rc == B._lib.B2B_EUNSUPPORTED
    rc = lib.b2b_chain_vjp_f64(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), None, D, N, D, D, D, None, 0, stream())
    assert rc == B._lib.B2B_EUNSUPPORTED and lib.b2b_last_launch_count() == 0
    torch.cuda.synchronize()
    assert torch.isnan(lj).all() and torch.isnan(xb).all()
    # at D = 8: slot 0 without μ is EINVAL, slots 2 / 3 EUNSUPPORTED, inverse / NULL L / not last EINVAL
    D = 8
    Lm = torch.eye(D, dtype=torch.float64, device="cuda")
    d.p1 = Lm.data_ptr()
    arr = (B._lib.LayerDesc64 * 1)(d)
    x = torch.zeros((N, D), dtype=torch.float64, device="cuda")
    xb = torch.empty((N, D), dtype=torch.float64, device="cuda")
    out = torch.empty(D * D, dtype=torch.float64, device="cuda")
    ws_b = lib.b2b_chain_vjp_workspace_bytes_f64(arr, 1, D, N)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    for slot, want in [(0, B._lib.B2B_EINVAL), (2, B._lib.B2B_EUNSUPPORTED), (3, B._lib.B2B_EUNSUPPORTED)]:
        ptrs = (ctypes.c_void_p * 4)()
        ptrs[slot] = out.data_ptr()
        rc = lib.b2b_chain_vjp_f64(arr, 1, x.data_ptr(), None, None, xb.data_ptr(), ctypes.cast(ptrs, ctypes.c_void_p), D, N,
                                   D, D, D, ws.data_ptr(), ws_b, stream())
        assert rc == want, (slot, rc)
    inv = B._lib.LayerDesc64()
    inv.kind, inv.inverse, inv.p1 = B._lib.MVNORMAL_TRIL, 1, Lm.data_ptr()
    nul = B._lib.LayerDesc64()
    nul.kind = B._lib.MVNORMAL_TRIL
    for descs in ([inv], [nul], [d, d]):
        a = (B._lib.LayerDesc64 * len(descs))(*descs)
        rc = lib.b2b_chain_run_f64(a, len(descs), x.data_ptr(), None, lj.data_ptr(), None, D, N, D, D, 0, None, 0, stream())
        assert rc == B._lib.B2B_EINVAL


def test_float64_rand_raises(B):
    import torch

    d = B.MvNormal(4, scale_tril=np.eye(4), dtype=torch.float64)
    with pytest.raises(TypeError):
        d.rand(8, seed=1)
