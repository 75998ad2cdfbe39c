"""Times the reverse-mode (VJP) path of the headline chain: 8 x PlanarLayer, D=128, N=2^20."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B

D, N, L = int(sys.argv[1]) if len(sys.argv) > 1 else 128, 1 << 20, int(sys.argv[2]) if len(sys.argv) > 2 else 8
rng = np.random.default_rng(0)
flow = B.Composed(*[B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                  (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                  rng.standard_normal(1).astype(np.float32)) for _ in range(L)])
x = B.from_numpy(rng.standard_normal((D, N)).astype(np.float32))
yb = B.from_numpy(rng.standard_normal((D, N)).astype(np.float32))
ljb = torch.randn(N, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for name, pg in (("xbar only", False), ("xbar + parameter cotangents", True)):
    ts = []
    for it in range(11):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        B.planar_chain_vjp(flow, x, yb, ljb, want_param_grads=pg)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    t = float(np.median(ts[3:]))
    # algorithmic bytes: main kernel reads x, ybar, ljbar and writes xbar + 3L scalars; the parameter pass re-reads
    # x, ybar and the scalars (twice: skinny reductions + S statistics)
    gb = 4.0 * N * (3 * D + 1 + 3 * L) / 1e9 + (4.0 * N * (2 * D + 6 * L) / 1e9 if pg else 0.0)
    print(f"{name:30s} D={D} L={L}  {t:.4f} ms  {N / t / 1e6:.2f} G samples/s  {gb / t * 1e3:.0f} GB/s "
          f"({gb / t * 1e3 / 3350.0 * 100:.1f} % of the 3350 GB/s H100 data sheet)")

# radial chain (BASELINE C3 shape: 6 layers, D = 64)
Dr, Lr = 64, 6
rflow = B.Composed(*[B.RadialLayer(rng.standard_normal(1).astype(np.float32), rng.standard_normal(1).astype(np.float32),
                                   rng.standard_normal(Dr).astype(np.float32)) for _ in range(Lr)])
xr = B.from_numpy(rng.standard_normal((Dr, N)).astype(np.float32))
ybr = B.from_numpy(rng.standard_normal((Dr, N)).astype(np.float32))
ts = []
for it in range(11):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    B.radial_chain_vjp(rflow, xr, ybr, ljb)
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
t = float(np.median(ts[3:]))
gb = 4.0 * N * (3 * Dr + 1) / 1e9
print(f"radial VJP (xbar + parameter cotangents) D={Dr} L={Lr}  {t:.4f} ms  {N / t / 1e6:.2f} G samples/s  {gb / t * 1e3:.0f} GB/s "
      f"({gb / t * 1e3 / 3350.0 * 100:.1f} % of the 3350 GB/s H100 data sheet)")


def timed(fn, reps=11):
    ts = []
    for it in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts[3:]))


# RQS (BASELINE C4 shape: K = 8 bins, D = 32; N = 2^20 here), both directions
Dq, K = 32, 8
spl = B.RationalQuadraticSpline(rng.standard_normal((Dq, K)).astype(np.float32), rng.standard_normal((Dq, K)).astype(np.float32),
                                rng.standard_normal((Dq, K - 1)).astype(np.float32), 3.0)
xq = B.from_numpy((rng.standard_normal((Dq, N)) * 1.5).astype(np.float32))
ybq = B.from_numpy(rng.standard_normal((Dq, N)).astype(np.float32))
for name, t_ in (("forward", spl), ("inverse", B.inverse(spl))):
    t = timed(lambda: B.rqs_vjp(t_, xq, ybq, ljb))
    gb = 4.0 * N * (3 * Dq + 1) / 1e9
    print(f"RQS VJP {name} D={Dq} K={K}  {t:.4f} ms  {N / t / 1e6:.2f} G samples/s  {gb / t * 1e3:.0f} GB/s "
          f"({gb / t * 1e3 / 3350.0 * 100:.1f} % of the 3350 GB/s H100 data sheet)")

# RealNVP layer kinds (BASELINE C5 shape: D = 256, n1 = n2 = 128; N = 2^19)
Dc, Nc = 256, 1 << 19
cl = B.Coupling(B.AffineConditioner((rng.standard_normal((256, 128)) * 0.02).astype(np.float32), np.zeros(256, np.float32)),
                B.PartitionMask(Dc, list(range(1, 129)), list(range(129, 257))))
bn = B.InvertibleBatchNorm(b=np.zeros(Dc, np.float32), logs=np.zeros(Dc, np.float32), m=np.zeros(Dc, np.float32), v=np.ones(Dc, np.float32))
xc = B.from_numpy(rng.standard_normal((Dc, Nc)).astype(np.float32))
ybc = B.from_numpy(rng.standard_normal((Dc, Nc)).astype(np.float32))
ljc = torch.randn(Nc, device="cuda")
gb = 4.0 * Nc * (3 * Dc + 1) / 1e9
for name, fn in (("coupling VJP", lambda: B.coupling_vjp(cl, xc, ybc, ljc)), ("batchnorm VJP", lambda: B.batchnorm_vjp(bn, xc, ybc, ljc))):
    t = timed(fn)
    print(f"{name} D={Dc} N=2^19  {t:.4f} ms  {Nc / t / 1e6:.2f} G samples/s  {gb / t * 1e3:.0f} GB/s "
          f"({gb / t * 1e3 / 3350.0 * 100:.1f} % of the 3350 GB/s H100 data sheet)")
