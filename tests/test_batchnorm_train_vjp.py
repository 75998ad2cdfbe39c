"""Reverse mode of the training-mode InvertibleBatchNorm (normalise.jl:51-67 with istraining() == true):
b2b_batchnorm_train_vjp_f32, interface.batchnorm_train_vjp, autograd.TrainingBatchNorm and RealNVP(batchnorm_training=True).

The float64 reference (tests/bn_train_vjp_oracle.py) is first pinned to central differences of
oracle_np.batchnorm_forward(training=True) on the CPU; the device results are then held to it with the parity gate of
tests/test_gpu_parity.py: 1e-5 norm-wise, widened only to twice the error of the float32 restatement on the same input."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle_np as O
import bn_train_vjp_oracle as BO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-5
f32 = np.float32


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-30))


def gate(o32, o64, k=2.0):
    return max(RTOL, k * rel(o32, o64))


def bn_params(D, rng, dtype=np.float64):
    b, logs = rng.standard_normal(D) * 0.3, rng.standard_normal(D) * 0.3
    m0, v0 = rng.standard_normal(D) * 0.1, rng.uniform(0.5, 1.5, D)
    return O.BatchNormParams(b.astype(dtype), logs.astype(dtype), m0.astype(dtype), v0.astype(dtype),
                             np.dtype(dtype).type(f32(1e-5)), np.dtype(dtype).type(f32(0.1)))


# ---- CPU: the oracle against finite differences -------------------------------------------------------------------------
def _objective(bn, x, ybar, ljbar):
    y, lj, _ = O.batchnorm_forward(bn, x, training=True)
    out = 0.0
    if ybar is not None:
        out += float((ybar * y).sum())
    if ljbar is not None:
        out += float((ljbar * lj).sum())
    return out


@pytest.mark.parametrize("case", ["ybar", "ljbar", "both", "constant_row"])
def test_oracle_matches_central_differences(case):
    rng = np.random.default_rng({"ybar": 1, "ljbar": 2, "both": 3, "constant_row": 4}[case])
    D, N = 4, 7
    bn = bn_params(D, rng)
    x = rng.standard_normal((D, N)) * 1.3 + 0.4
    if case == "constant_row":
        x[2] = 0.7  # v = 0 on that row: σ² = eps
    ybar = None if case == "ljbar" else rng.standard_normal((D, N))
    ljbar = None if case == "ybar" else rng.standard_normal(N)
    xbar, bbar, logsbar = BO.batchnorm_train_vjp(bn, x, ybar, ljbar)
    h = 1e-6 if case != "constant_row" else 1e-9
    fd = np.zeros_like(x)
    for i in range(D):
        for j in range(N):
            xp, xm = x.copy(), x.copy()
            xp[i, j] += h
            xm[i, j] -= h
            fd[i, j] = (_objective(bn, xp, ybar, ljbar) - _objective(bn, xm, ybar, ljbar)) / (2 * h)
    assert rel(xbar, fd) <= 1e-6, rel(xbar, fd)
    for field, got in (("b", bbar), ("logs", logsbar)):
        g = np.zeros(D)
        for i in range(D):
            bp, bm = (O.BatchNormParams(**{**bn.__dict__, field: getattr(bn, field).copy()}) for _ in range(2))
            getattr(bp, field)[i] += 1e-6
            getattr(bm, field)[i] -= 1e-6
            g[i] = (_objective(bp, x, ybar, ljbar) - _objective(bm, x, ybar, ljbar)) / 2e-6
        assert rel(got, g) <= 1e-6 or np.abs(got - g).max() <= 1e-8, (field, got, g)
    if case == "ljbar":  # the variance-through-logjac term is the whole of x̄ here
        assert np.linalg.norm(xbar) > 1e-3


def test_oracle_column_shards_add_up():
    """With the full batch's statistics, the shards' x̄ are the full x̄'s columns and their b̄ / l̄ogs sum to the full ones
    (the per-rank meaning of the device call's parameter cotangents)."""
    rng = np.random.default_rng(5)
    D, N = 6, 101
    bn = bn_params(D, rng)
    x, ybar, ljbar = rng.standard_normal((D, N)) * 2 - 1, rng.standard_normal((D, N)), rng.standard_normal(N)
    xo, bo, lo = BO.batchnorm_train_vjp(bn, x, ybar, ljbar)
    cuts = [0, 17, 60, N]
    bsum, lsum = np.zeros(D), np.zeros(D)
    for lo_, hi_ in zip(cuts[:-1], cuts[1:]):
        xs, bs, ls = BO.batchnorm_train_vjp_shard(bn, x, ybar, ljbar, lo_, hi_)
        assert np.array_equal(xs, xo[:, lo_:hi_])
        bsum += bs
        lsum += ls
    assert np.allclose(bsum, bo, rtol=1e-12, atol=1e-12) and np.allclose(lsum, lo, rtol=1e-12, atol=1e-12)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def _inputs(D, N, rng, offset="affine"):
    x = rng.standard_normal((D, N), dtype=np.float32)
    x = (x * f32(1.7) + f32(0.3)) if offset == "affine" else (x + f32(50.0))
    return x.astype(f32), rng.standard_normal((D, N), dtype=np.float32), rng.standard_normal(N, dtype=np.float32)


def _check(B, bn32, x, ybar, ljbar, xbar, bbar, lbar):
    bn64 = O.BatchNormParams(*(np.asarray(getattr(bn32, f), np.float64) for f in ("b", "logs", "m", "v")),
                             np.float64(bn32.eps), np.float64(bn32.mtm))
    up = lambda a: None if a is None else a.astype(np.float64)
    xo, bo, lo = BO.batchnorm_train_vjp(bn64, x.astype(np.float64), up(ybar), up(ljbar))
    x32, _, _ = BO.batchnorm_train_vjp(bn32, x, ybar, ljbar)
    N = x.shape[1]
    assert rel(xbar, xo) <= gate(x32, xo), (rel(xbar, xo), rel(x32, xo))
    for got, want in ((bbar, bo), (lbar, lo)):
        assert np.all(np.abs(np.asarray(got, np.float64) - want) <= 2e-5 * np.maximum(np.abs(want), np.sqrt(N))), \
            np.abs(np.asarray(got, np.float64) - want).max()


def _layer(B, D, rng):
    b, logs = (rng.standard_normal(D) * 0.3).astype(f32), (rng.standard_normal(D) * 0.3).astype(f32)
    m0, v0 = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    bn = B.InvertibleBatchNorm(b=b, logs=logs, m=m0, v=v0, training=True)
    return bn, O.BatchNormParams(b, logs, m0, v0, f32(1e-5), f32(0.1))


@pytest.mark.gpu
@pytest.mark.parametrize("N", [2, 5, 1000, 65539])
@pytest.mark.parametrize("D", [3, 10, 32, 64, 128, 200, 256, 777, 1024])
def test_parity_with_the_oracle(B, D, N):
    import torch

    rng = np.random.default_rng(1000 * D + N)
    bn, bn32 = _layer(B, D, rng)
    x, ybar, ljbar = _inputs(D, N, rng)
    m0, v0 = bn.m.clone(), bn.v.clone()
    xbar, g = B.batchnorm_train_vjp(bn, B.from_numpy(x), B.from_numpy(ybar), torch.as_tensor(ljbar, device="cuda"))
    _check(B, bn32, x, ybar, ljbar, B.to_numpy(xbar), B.to_numpy(g["b"]), B.to_numpy(g["logs"]))
    assert torch.equal(bn.m, m0) and torch.equal(bn.v, v0)  # the moving statistics are not touched


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ybar_none", "ljbar_none", "padded_ld", "misaligned", "offset50", "in_place"])
@pytest.mark.parametrize("D", [3, 64, 200, 1024])
def test_cotangent_and_layout_variants(B, D, variant):
    import torch

    rng = np.random.default_rng(7 * D + len(variant))
    N = 4097
    bn, bn32 = _layer(B, D, rng)
    x, ybar, ljbar = _inputs(D, N, rng, "offset50" if variant == "offset50" else "affine")
    yb = None if variant == "ybar_none" else ybar
    lb = None if variant == "ljbar_none" else ljbar
    L_ = B._lib.lib()
    nbytes = L_.b2b_batchnorm_train_vjp_workspace_bytes(D)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    bbar, lbar = torch.empty(D, device="cuda"), torch.empty(D, device="cuda")
    pad = 3 if variant == "padded_ld" else 0

    def place(a, off=0):  # (D, N) column-major with leading dimension D + pad, base offset by `off` floats
        flat = torch.full(((D + pad) * N + off,), 7.0, device="cuda")
        v = flat[off:].view(N, D + pad)[:, :D].t()
        if a is not None:
            v.copy_(B.from_numpy(a))
        return flat, v

    off = 1 if variant == "misaligned" else 0
    _, xd = place(x, off)
    ybuf, yd = place(yb, off) if yb is not None else (None, None)
    lbd = torch.as_tensor(lb, device="cuda") if lb is not None else None
    if variant == "in_place":
        xbuf, xbd = ybuf, yd
    else:
        xbuf, xbd = place(None, off)
    rc = L_.b2b_batchnorm_train_vjp_f32(xd.data_ptr(), yd.data_ptr() if yd is not None else None,
                                        lbd.data_ptr() if lbd is not None else None, xbd.data_ptr(), bbar.data_ptr(),
                                        lbar.data_ptr(), bn.logs.data_ptr(), bn.eps, D, N, D + pad, D + pad, D + pad, None,
                                        ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    _check(B, bn32, x, yb, lb, B.to_numpy(xbd), B.to_numpy(bbar), B.to_numpy(lbar))
    if pad:
        assert bool((xbuf.view(N, D + pad)[:, D:] == 7.0).all()), "padding between columns was overwritten"


def _raw_call(B, x, ybar, ljbar, xbar, bbar, lbar, logs, D, N, ws, nbytes, ld=None, eps=1e-5):
    import torch

    ptr = lambda t: t.data_ptr() if t is not None else None
    ld = D if ld is None else ld
    return B._lib.lib().b2b_batchnorm_train_vjp_f32(ptr(x), ptr(ybar), ptr(ljbar), ptr(xbar), ptr(bbar), ptr(lbar), ptr(logs),
                                                    eps, D, N, ld, ld, ld, None, ptr(ws), nbytes,
                                                    torch.cuda.current_stream().cuda_stream)


@pytest.mark.gpu
def test_deterministic_and_graph_replay_is_bit_identical(B):
    import torch

    rng = np.random.default_rng(11)
    D, N = 256, 100_003
    bn, _ = _layer(B, D, rng)
    x, ybar, ljbar = _inputs(D, N, rng)
    xd, yd, ld = B.from_numpy(x), B.from_numpy(ybar), torch.as_tensor(ljbar, device="cuda")
    a, ga = B.batchnorm_train_vjp(bn, xd, yd, ld)
    b, gb = B.batchnorm_train_vjp(bn, xd, yd, ld)
    assert torch.equal(a, b) and torch.equal(ga["b"], gb["b"]) and torch.equal(ga["logs"], gb["logs"])
    nbytes = B._lib.lib().b2b_batchnorm_train_vjp_workspace_bytes(D)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    xb, bb, lb = B.colmajor_empty(D, N), torch.empty(D, device="cuda"), torch.empty(D, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        assert _raw_call(B, xd, yd, ld, xb, bb, lb, bn.logs, D, N, ws, nbytes) == 0
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        rc = _raw_call(B, xd, yd, ld, xb, bb, lb, bn.logs, D, N, ws, nbytes)
    assert rc == 0
    xb.fill_(0.0)
    bb.fill_(0.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(xb, a) and torch.equal(bb, ga["b"]) and torch.equal(lb, ga["logs"])


@pytest.mark.gpu
def test_training_module_moves_the_statistics_once(B):
    import torch

    rng = np.random.default_rng(12)
    D, N = 96, 5000
    layer = B.autograd.TrainingBatchNorm(D)
    with torch.no_grad():
        layer.b.copy_(torch.as_tensor(rng.standard_normal(D) * 0.2, dtype=torch.float32))
        layer.logs.copy_(torch.as_tensor(rng.standard_normal(D) * 0.2, dtype=torch.float32))
    x, ybar, ljbar = _inputs(D, N, rng)
    xt = B.from_numpy(x).requires_grad_(True)
    y, lj = layer(xt)
    ((y * B.from_numpy(ybar)).sum() + (lj * torch.as_tensor(ljbar, device="cuda")).sum()).backward()
    bn64 = O.BatchNormParams(layer.b.detach().double().cpu().numpy(), layer.logs.detach().double().cpu().numpy(),
                             np.zeros(D), np.ones(D), np.float64(f32(1e-5)), np.float64(f32(0.1)))
    yo, ljo, (m1, v1) = O.batchnorm_forward(bn64, x.astype(np.float64), training=True)
    assert rel(B.to_numpy(y.detach()), yo) <= RTOL and rel(B.to_numpy(lj.detach()), ljo) <= RTOL
    assert rel(B.to_numpy(layer.m), m1) <= RTOL and rel(B.to_numpy(layer.v), v1) <= RTOL  # updated once, not twice
    xo, bo, lo = BO.batchnorm_train_vjp(bn64, x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64))
    assert rel(B.to_numpy(xt.grad), xo) <= RTOL
    assert rel(B.to_numpy(layer.b.grad), bo) <= 2e-5 and rel(B.to_numpy(layer.logs.grad), lo) <= 2e-5


@pytest.mark.gpu
def test_status_codes(B):
    import torch

    L_ = B._lib.lib()
    assert L_.b2b_batchnorm_train_vjp_workspace_bytes(0) == 0 and L_.b2b_batchnorm_train_vjp_workspace_bytes(1025) == 0
    assert L_.b2b_batchnorm_train_vjp_workspace_bytes(1024) > 0
    D, N = 1025, 64
    x, yb = torch.randn(N, D, device="cuda").t(), torch.randn(N, D, device="cuda").t()
    xb = torch.full((N, D), 7.0, device="cuda").t()
    logs, bb, lb = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    ws = torch.empty((1 << 20,), dtype=torch.uint8, device="cuda")
    assert _raw_call(B, x, yb, None, xb, bb, lb, logs, D, N, ws, ws.numel()) == B._lib.B2B_EUNSUPPORTED
    torch.cuda.synchronize()
    assert bool((xb == 7.0).all())
    D = 64
    nbytes = L_.b2b_batchnorm_train_vjp_workspace_bytes(D)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    ybase = torch.randn(N, D, device="cuda")
    x, yb, xb = torch.randn(N, D, device="cuda").t(), ybase.t(), B.colmajor_empty(D, N)
    logs, bb, lb = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    EINVAL = B._lib.B2B_EINVAL
    for n in (0, 1):
        assert _raw_call(B, x, yb, None, xb, bb, lb, logs, D, n, ws, nbytes) == EINVAL
    assert _raw_call(B, None, yb, None, xb, bb, lb, logs, D, N, ws, nbytes) == EINVAL
    assert _raw_call(B, x, yb, None, None, bb, lb, logs, D, N, ws, nbytes) == EINVAL
    assert _raw_call(B, x, yb, None, xb, bb, lb, None, D, N, ws, nbytes) == EINVAL
    assert _raw_call(B, x, yb, None, xb, bb, None, logs, D, N, ws, nbytes) == EINVAL
    assert _raw_call(B, x, yb, None, xb, None, lb, logs, D, N, ws, nbytes) == EINVAL
    shifted = ybase.reshape(-1)[D:].view(N - 1, D).t()  # overlaps ybar one column later
    assert _raw_call(B, x, yb, None, shifted, bb, lb, logs, D, N - 1, ws, nbytes) == EINVAL
    assert _raw_call(B, x, yb, None, x, bb, lb, logs, D, N, ws, nbytes) == EINVAL  # x̄ over x
    assert _raw_call(B, x, yb, None, xb, bb, lb, logs, D, N, ws, nbytes - 1) == B._lib.B2B_EWORKSPACE
    assert _raw_call(B, x, yb, None, xb, None, None, logs, D, N, ws, nbytes) == 0  # no parameter cotangents
    assert _raw_call(B, x, yb, None, yb, bb, lb, logs, D, N, ws, nbytes) == 0  # x̄ exactly over ȳ
    torch.cuda.synchronize()


def _realnvp_oracle(flow, x, ybar, ljbar):
    """Float64 chain: coupling_affine_forward + batchnorm_forward(training=True) per block, then coupling_affine_vjp and
    the training-mode BatchNorm VJP layer by layer, last to first."""
    D = flow.dims
    h = D // 2
    inputs, params = [], []
    z = x
    for l in range(len(flow.W)):
        first = l % 2 == 0
        idx1 = list(range(1, h + 1)) if first else list(range(h + 1, D + 1))
        idx2 = list(range(h + 1, D + 1)) if first else list(range(1, h + 1))
        W, c = flow.W[l].detach().double().cpu().numpy(), flow.c[l].detach().double().cpu().numpy()
        bn = O.BatchNormParams(flow.b[l].detach().double().cpu().numpy(), flow.logs[l].detach().double().cpu().numpy(),
                               np.zeros(D), np.ones(D), np.float64(f32(1e-5)), np.float64(f32(0.1)))
        u, _ = O.coupling_affine_forward(idx1, idx2, W, c, z)
        inputs.append((z, u))
        params.append((idx1, idx2, W, c, bn))
        z, _, _ = O.batchnorm_forward(bn, u, training=True)
    grads = [None] * len(params)
    cot = ybar
    for l in reversed(range(len(params))):
        idx1, idx2, W, c, bn = params[l]
        zin, u = inputs[l]
        ubar, bb, lb = BO.batchnorm_train_vjp(bn, u, cot, ljbar)
        cot, Wb, cb = O.coupling_affine_vjp(idx1, idx2, W, c, zin, ubar, ljbar)
        grads[l] = (Wb, cb, bb, lb)
    return cot, grads


@pytest.mark.gpu
def test_realnvp_with_training_batchnorm_gradients(B):
    import torch

    rng = np.random.default_rng(13)
    D, N = 64, 4096
    flow = B.autograd.RealNVP(D, 3, generator=torch.Generator().manual_seed(0), batchnorm_training=True)
    with torch.no_grad():
        for l in range(3):
            flow.c[l].copy_(torch.as_tensor(rng.standard_normal(flow.c[l].numel()) * 0.1, dtype=torch.float32))
            flow.b[l].copy_(torch.as_tensor(rng.standard_normal(D) * 0.2, dtype=torch.float32))
            flow.logs[l].copy_(torch.as_tensor(rng.standard_normal(D) * 0.2, dtype=torch.float32))
    x, ybar, ljbar = _inputs(D, N, rng)
    xt = B.from_numpy(x).requires_grad_(True)
    y, lj = flow(xt)
    ((y * B.from_numpy(ybar)).sum() + (lj * torch.as_tensor(ljbar, device="cuda")).sum()).backward()
    xo, go = _realnvp_oracle(flow, x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64))
    assert rel(B.to_numpy(xt.grad), xo) <= 5e-5, rel(B.to_numpy(xt.grad), xo)
    for l in range(3):
        for got, want in zip((flow.W[l].grad, flow.c[l].grad, flow.b[l].grad, flow.logs[l].grad), go[l]):
            assert rel(got.cpu().numpy(), want) <= 5e-5, (l, rel(got.cpu().numpy(), want))
    with pytest.raises(AssertionError, match="test mode"):
        flow.inverse(y.detach())
    with pytest.raises(AssertionError, match="test mode"):
        flow.nll(y.detach())


@pytest.mark.gpu
def test_variational_inference_lowers_the_reverse_kl(B):
    """Turing's use of a flow: q = flow(MvNormal(0, I)) fitted to a diagonal Gaussian p by minimising a Monte-Carlo
    estimate of KL(q‖p) = E_z[log N(z) − logjac − log p(flow(z))], with z from the in-kernel Philox sampler."""
    import torch

    D, N = 8, 4096
    flow = B.autograd.RealNVP(D, 2, generator=torch.Generator().manual_seed(1), batchnorm_training=True)
    base = B.MvNormal(D)
    mu = torch.linspace(-1.0, 2.0, D, device="cuda")[:, None]
    sig = torch.linspace(0.5, 1.5, D, device="cuda")[:, None]
    opt = torch.optim.Adam(flow.parameters(), lr=2e-2)
    c = 0.5 * D * float(np.log(2 * np.pi))
    losses = []
    for step in range(80):
        z = base.rand(N, seed=step)
        x, lj = flow(z)
        logq0 = -0.5 * (z * z).sum(0) - c
        logp = -0.5 * (((x - mu) / sig) ** 2).sum(0) - torch.log(sig).sum() - c
        loss = (logq0 - lj - logp).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    start, end = np.mean(losses[:5]), np.mean(losses[-5:])
    assert np.isfinite(losses).all() and end < 0.1 * start, (start, end)


@pytest.mark.gpu
def test_sharded_over_two_gpus():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "mgpu_bn_train_vjp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "bn train vjp ok" in r.stdout
