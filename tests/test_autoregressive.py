"""GPU tests of the masked autoregressive layer, B2B_AUTOREGRESSIVE_MLP: MaskedAutoregressive (MAF / IAF with a MADE
conditioner) against the float64 reference of tests/autoregressive_oracle.py.  Gates are tied to the reference's own
float32 error on the same input, as in test_gpu_parity.gate: max(1e-5, 2 × ‖oracle32 − oracle64‖ / ‖oracle64‖),
norm-wise."""
import numpy as np
import pytest

import autoregressive_oracle as A
import chain_vjp_oracle as V
import rsample_oracle as R
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
f32 = np.float32
RTOL = 1e-5
ACTS = [("tanh", 0.0), ("leaky_relu", 0.1)]


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


def spec(rng, D, H, with_c=True, deg="default", scale=0.8):
    """(W1, c1, W2, c2, degrees) with the weights scaled so that s stays O(1)."""
    W1 = (rng.standard_normal((H, D)) * scale / np.sqrt(D)).astype(f32)
    W2 = (rng.standard_normal((2 * D, H)) * scale / np.sqrt(H)).astype(f32)
    c1 = (rng.standard_normal(H) * 0.3).astype(f32) if with_c else None
    c2 = (rng.standard_normal(2 * D) * 0.2).astype(f32) if with_c else None
    m = A.default_degrees(D, H) if deg == "default" else rng.integers(-1, D + 2, H)
    return W1, c1, W2, c2, m


def layer(B, sp, act="tanh", slope=0.0):
    return B.MaskedAutoregressive(*sp[:4], degrees=sp[4], activation=act, slope=slope)


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
@pytest.mark.parametrize("H", [1, 32, 100, 256])
@pytest.mark.parametrize("D", [1, 2, 7, 64, 128])
def test_parity(B, D, H, act, slope, inv):
    rng = np.random.default_rng(D * 7 + H + inv)
    with_c = (D + H) % 2 == 0
    N = 200 if with_c else 67  # 67: not a multiple of the tile
    sp = spec(rng, D, H, with_c, deg="default" if H % 2 == 0 else "random")
    x = rng.standard_normal((D, N)).astype(f32)
    lay = layer(B, sp, act, slope)
    y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, B.from_numpy(x))
    f = A.inverse if inv else A.forward
    y64, l64 = f(*sp, act, slope, x.astype(np.float64))
    y32, l32 = f(*sp, act, slope, x, f32)
    gate(B.to_numpy(y), y64, y32, "y")
    gate(B.to_numpy(lj), l64, l32, "logjac")
    # in place: the same bits
    xd = B.from_numpy(x)
    y2, lj2 = B.with_logabsdet_jacobian_(B.inverse(lay) if inv else lay, xd)
    assert B.to_numpy(xd).tobytes() == B.to_numpy(y).tobytes()
    assert B.to_numpy(lj2).tobytes() == B.to_numpy(lj).tobytes()


@pytest.mark.parametrize("act,slope", ACTS)
@pytest.mark.parametrize("D,H", [(3, 8), (64, 100), (128, 256)])
def test_round_trip(B, D, H, act, slope):
    rng = np.random.default_rng(D + H)
    sp = spec(rng, D, H)
    x = rng.standard_normal((D, 1000)).astype(f32)
    lay = layer(B, sp, act, slope)
    y, lj = B.with_logabsdet_jacobian(lay, B.from_numpy(x))
    xr, ljr = B.with_logabsdet_jacobian(B.inverse(lay), y)
    assert rel(B.to_numpy(xr), x) < 1e-5
    assert rel(B.to_numpy(ljr), -B.to_numpy(lj)) < 1e-5


@pytest.mark.parametrize("inv", [False, True])
def test_masked_entries_are_not_read(B, inv):
    rng = np.random.default_rng(5 + inv)
    D, H, N = 20, 48, 333
    sp = spec(rng, D, H, deg="random")
    M1, M2 = A.masks(sp[4], D)
    W1n, W2n = sp[0].copy(), sp[2].copy()
    W1n[~M1], W2n[~M2] = np.nan, np.nan
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    outs = []
    for W1, W2 in ((sp[0], sp[2]), (W1n, W2n)):
        lay = B.MaskedAutoregressive(W1, sp[1], W2, sp[3], degrees=sp[4])
        y, lj = B.with_logabsdet_jacobian(B.inverse(lay) if inv else lay, x)
        outs.append((B.to_numpy(y).tobytes(), B.to_numpy(lj).tobytes()))
    assert outs[0] == outs[1]


@pytest.mark.parametrize("inv", [False, True])
def test_autoregressive_property(B, inv):
    """Perturbing row j changes no output row i < j, bit for bit."""
    rng = np.random.default_rng(9 + inv)
    D, H, N = 24, 64, 100
    sp = spec(rng, D, H, deg="random")
    lay = layer(B, sp)
    t = B.inverse(lay) if inv else lay
    x = rng.standard_normal((D, N)).astype(f32)
    y0 = B.to_numpy(B.transform(t, B.from_numpy(x)))
    for j in (0, 5, D - 1):
        xp = x.copy()
        xp[j] += 0.5
        y1 = B.to_numpy(B.transform(t, B.from_numpy(xp)))
        assert y1[:j].tobytes() == y0[:j].tobytes()
        assert not np.array_equal(y1[j], y0[j])


@pytest.mark.parametrize("inv", [False, True])
@pytest.mark.parametrize("act,slope", ACTS)
@pytest.mark.parametrize("D,H,N,with_c,cots", [
    (1, 1, 300, True, "yl"), (7, 32, 777, False, "yl"), (40, 100, 1500, True, "y"), (64, 64, 500, True, "l"),
    (128, 256, 300, True, "yl")])
def test_vjp(B, D, H, N, with_c, cots, act, slope, inv):
    import torch

    rng = np.random.default_rng(D + 3 * H + N + inv)
    sp = spec(rng, D, H, with_c, deg="random")
    x = rng.standard_normal((D, N)).astype(f32)
    yb = rng.standard_normal((D, N)).astype(f32) if "y" in cots else None
    lb = rng.standard_normal(N).astype(f32) if "l" in cots else None
    t = B.inverse(layer(B, sp, act, slope)) if inv else layer(B, sp, act, slope)

    def run():
        return B.chain_vjp(t, B.from_numpy(x), None if yb is None else B.from_numpy(yb),
                           None if lb is None else torch.from_numpy(lb).cuda())

    xbar, grads = run()
    xb64, g64 = A.vjp(*sp, act, slope, x, yb, lb, inverse=inv)
    xb32, g32 = A.vjp(*sp, act, slope, x, yb, lb, inverse=inv, dtype=f32)
    gate(B.to_numpy(xbar), xb64, xb32, "xbar")
    names = ("W1", "c1", "W2", "c2") if with_c else ("W1", "W2")
    assert set(grads[0]) == set(names)
    M1, M2 = A.masks(sp[4], D)
    for k in names:
        got = grads[0][k].cpu().numpy()
        gate(got, g64[k], g32[k], k + "bar")
    assert not grads[0]["W1"].cpu().numpy()[~M1].any() and not grads[0]["W2"].cpu().numpy()[~M2].any()
    xbar2, grads2 = run()  # deterministic
    assert B.to_numpy(xbar2).tobytes() == B.to_numpy(xbar).tobytes()
    for k in names:
        assert grads2[0][k].cpu().numpy().tobytes() == grads[0][k].cpu().numpy().tobytes()


def _maf(B, rng, D, H=24):
    """inverse(A₃) ∘ Permute ∘ BatchNorm ∘ inverse(A₂) ∘ Permute ∘ MLP coupling ∘ inverse(A₁), device and oracle layers
    (oracle layers as (layer, inverse flag) in application order)."""
    import coupling_mlp_oracle as M

    dev, ora = [], []

    def ar(act):
        sp = spec(rng, D, H, deg="random", scale=0.5)
        dev.append(B.inverse(layer(B, sp, *act)))
        ora.append((A.AutoregressiveLayer(*sp, *act), True))

    def perm():
        p = rng.permutation(D) + 1
        dev.append(B.Permute(p))
        ora.append((O.Layer("permute", dict(A=O.permute_matrix_from_indices(p))), False))

    ar(("tanh", 0.0))
    i1, i2 = [int(i) for i in range(1, D // 2 + 1)], [int(i) for i in range(D // 2 + 1, D + 1)]
    W1 = (rng.standard_normal((H, len(i2))) * 0.3).astype(f32)
    W2 = (rng.standard_normal((2 * len(i1), H)) * 0.1).astype(f32)
    c1, c2 = (rng.standard_normal(H) * 0.1).astype(f32), (rng.standard_normal(2 * len(i1)) * 0.1).astype(f32)
    dev.append(B.Coupling(B.MLPConditioner(W1, c1, W2, c2), B.PartitionMask(D, i1, i2)))
    ora.append((M.MLPLayer(i1, i2, W1, c1, W2, c2), False))
    perm()
    ar(("leaky_relu", 0.2))
    b, logs = (rng.standard_normal(D) * 0.1).astype(f32), (rng.standard_normal(D) * 0.1).astype(f32)
    m, v = (rng.standard_normal(D) * 0.1).astype(f32), rng.uniform(0.5, 1.5, D).astype(f32)
    dev.append(B.InvertibleBatchNorm(b=b, logs=logs, m=m, v=v))
    ora.append((O.Layer("batchnorm", dict(bn=O.BatchNormParams(b=b, logs=logs, m=m, v=v, eps=1e-5))), False))
    perm()
    ar(("tanh", 0.0))
    return B.Composed(*dev), ora


def _run(ora, x, dt, inverse=False):
    cur, lj = np.asarray(x, dt), 0.0
    seq = [(lay, not f) for lay, f in reversed(ora)] if inverse else ora
    for lay, f in seq:
        cur, l = (lay.inverse if f else lay.forward)(cur)
        lj = lj + l
    return cur, lj


def test_maf_logpdf_vjp_and_rand(B):
    import torch

    rng = np.random.default_rng(31)
    D, N = 16, 600
    flow, ora = _maf(B, rng, D)
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.3, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu=mu, sigma=sigma), flow)
    y = rng.standard_normal((D, N)).astype(f32)
    yd = B.from_numpy(y)
    lp = B.to_numpy(B.logpdf(td, yd))

    def chain_lp(dt):
        x, lj = _run(ora, y, dt, inverse=True)
        return O.mvnormal_diag_logpdf(mu.astype(dt), sigma.astype(dt), x) + lj

    lp64, lp32 = chain_lp(np.float64), chain_lp(f32)
    gate(lp, lp64, lp32, "logpdf")
    s, lps = B.logpdf_sum(td, yd)
    assert B.to_numpy(lps).tobytes() == lp.tobytes()
    assert abs(float(s) - lp64.sum()) <= 1e-4 * abs(lp64.sum()) + 1e-3
    lb = rng.standard_normal(N)
    ybar, fgrads, _ = B.logpdf_vjp(td, yd, torch.from_numpy(lb.astype(f32)).cuda())
    inv_layers = [lay for lay, _ in reversed(ora)]
    flags = [not f for _, f in reversed(ora)]
    g, grads, _ = V.chain_vjp(inv_layers, flags, y, None, lb, mu, sigma, terminal=True)
    assert rel(B.to_numpy(ybar), g) < 1e-4
    flow_grads = grads[::-1]
    for k in (0, 3, 6):
        for name in ("W1", "c1", "W2", "c2"):
            assert rel(fgrads[k][name].cpu().numpy(), flow_grads[k][name]) < 1e-4, (k, name)
    # rand runs the sequential direction of every layer
    ys, ljs = B.rand(td, 3001, seed=77, offset=2, with_logjac=True)
    x = B.to_numpy(B.rand(td.dist, 3001, seed=77, offset=2))
    y64, l64 = _run(ora, x.astype(np.float64), np.float64)
    y32, l32 = _run(ora, x, f32)
    gate(B.to_numpy(ys), y64, y32, "rand y")
    gate(B.to_numpy(ljs), l64, l32, "rand logjac")


def test_iaf_rand_logpdf_and_rand_vjp(B):
    import torch

    rng = np.random.default_rng(41)
    D, N, H, SEED = 12, 4000, 32, 1234
    dev, ora = [], []
    for k in range(3):
        sp = spec(rng, D, H, scale=0.5)
        dev.append(layer(B, sp, *ACTS[k % 2]))
        ora.append(A.AutoregressiveLayer(*sp, *ACTS[k % 2]))
        if k < 2:
            p = rng.permutation(D) + 1
            dev.append(B.Permute(p))
            ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(p))))
    mu, sigma = (rng.standard_normal(D) * 0.2).astype(f32), rng.uniform(0.7, 1.3, D).astype(f32)
    td = B.transformed(B.MvNormal(D, mu=mu, sigma=sigma), B.Composed(*dev))
    z = O.philox_normals(SEED, 0, D, N)
    x = B.to_numpy(B.rand(td.dist, N, seed=SEED))
    y, lq = B.rand_logpdf(td, N, seed=SEED)
    y64, lj64 = O.chain_forward(ora, x.astype(np.float64))
    y32, lj32 = O.chain_forward(ora, x)
    gate(B.to_numpy(y), y64, y32, "y")
    lq64 = O.mvnormal_diag_logpdf(mu, sigma, x.astype(np.float64)) - lj64
    assert rel(B.to_numpy(lq), lq64) < 1e-5
    ybar = rng.standard_normal((D, N)).astype(f32)
    qbar = rng.standard_normal(N).astype(f32)
    fg, bg = B.rand_vjp(td, N, B.from_numpy(ybar), torch.from_numpy(qbar).cuda(), seed=SEED)
    g64, b64 = R.vjp(ora, [False] * len(ora), z, ybar, qbar, mu, sigma, x=x)
    for k in (0, 2, 4):
        for name in ("W1", "c1", "W2", "c2"):
            assert rel(fg[k][name].cpu().numpy(), g64[k][name]) < 2e-4, (k, name)
    assert rel(bg["μ"].cpu().numpy(), b64["μ"]) < 2e-4 and rel(bg["σ"].cpu().numpy(), b64["σ"]) < 2e-4


@pytest.mark.parametrize("kind", ["maf", "iaf"])
def test_flow_training(B, kind):
    """A 3-layer MAF trained by NLL on seeded data, or a 3-layer IAF by the reparameterised ELBO of a 2-D target: the
    first gradient matches the float64 oracle and the loss goes down."""
    import torch

    rng = np.random.default_rng(81)
    D, N, H = 4, 4096, 16
    dev, ora = [], []
    for k in range(3):
        sp = spec(rng, D, H, scale=0.3)
        dev.append(layer(B, sp, *ACTS[k % 2]))
        ora.append(A.AutoregressiveLayer(*sp, *ACTS[k % 2]))
        if k < 2:
            p = np.roll(np.arange(1, D + 1), 1)
            dev.append(B.Permute(p))
            ora.append(O.Layer("permute", dict(A=O.permute_matrix_from_indices(p))))
    if kind == "maf":
        flow = B.autograd.Flow(B.Composed(*[B.inverse(t) for t in dev]))
        z = rng.standard_normal((D, N))
        data = np.stack([z[0] * 1.5, z[1] * 0.5 + 0.3 * z[0] ** 2] + [z[j] * (0.5 + 0.1 * j) for j in range(2, D)])
        data = data.astype(f32)
        y = B.from_numpy(data)
        loss = flow.nll(y)
        loss.backward()
        inv_layers = ora[::-1]  # logpdf runs inverse(flow): every layer of `ora` forward, the last first
        flags = [False] * len(inv_layers)
        g, grads, _ = V.chain_vjp(inv_layers, flags, data, None, -np.ones(N), np.zeros(D), np.ones(D), terminal=True)
        x, lj = _run(list(zip(inv_layers, flags)), data.astype(np.float64), np.float64)
        lp = O.mvnormal_diag_logpdf(None, None, x) + lj
        assert abs(float(loss.detach()) + lp.sum()) <= 1e-4 * abs(lp.sum())
        grads = grads[::-1]
        step = lambda: flow.nll(y)  # noqa: E731
    else:
        flow = B.autograd.Flow(B.Composed(*dev), B.MvNormal(D))
        SEED = 5

        def elbo_loss():
            ys, lq = flow.rsample(N, seed=SEED)
            logp = -0.5 * ((ys[0] / 2) ** 2 + ((ys[1] - 0.5 * ys[0] ** 2) / 0.5) ** 2) - 0.5 * (ys[2:] ** 2).sum(0)
            return (lq - logp).mean()

        loss = elbo_loss()
        loss.backward()
        zz = O.philox_normals(SEED, 0, D, N)
        xx = B.to_numpy(B.rand(B.MvNormal(D), N, seed=SEED))
        ys, _ = O.chain_forward(ora, xx.astype(np.float64))
        ybar = np.zeros((D, N))
        ybar[0] = (ys[0] / 4 - ys[0] * (ys[1] - 0.5 * ys[0] ** 2) / 0.25) / N
        ybar[1] = ((ys[1] - 0.5 * ys[0] ** 2) / 0.25) / N
        ybar[2:] = ys[2:] / N
        grads, _ = R.vjp(ora, [False] * len(ora), zz, ybar, np.full(N, 1.0 / N), x=xx)
        step = elbo_loss
    ps = list(flow.params)
    for k, gk in zip(range(3), grads[::2]):
        for i, name in enumerate(("W1", "c1", "W2", "c2")):
            got = ps[4 * k + i].grad.cpu().numpy()
            assert rel(got.T if got.ndim == 2 else got, gk[name]) < 1e-4, (kind, k, name)
    opt = torch.optim.Adam(flow.parameters(), lr=1e-2)
    first = float(loss.detach())
    for _ in range(30):
        opt.zero_grad()
        loss = step()
        loss.backward()
        opt.step()
    assert float(step().detach()) < first - 0.01 * abs(first)
