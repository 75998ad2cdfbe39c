"""Times the reverse-mode (VJP) path of the headline chain: 8 x PlanarLayer, D=128, N=2^20.
`python tools/bench_vjp.py chain` times b2b_chain_vjp_f32 instead, as device time of graph-captured calls: (a) the
elementwise-run kernel alone on Stacked(Logit + exp rows) + Permute + MvNormal, (b) the logpdf gradient of
inverse(8 x Planar) + MvNormal through logpdf_vjp against planar_chain_vjp with the base density's cotangent in torch, the
two routes alternated.  `python tools/bench_vjp.py chain64` times b2b_chain_vjp_f64 on the Float64 8 x Planar chain at D=128,
N=2^16 (x̄ and every parameter cotangent), also as device time of graph-captured calls."""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B


def print_card():
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(f"card: {torch.cuda.get_device_name()}, power limit: {power}")


def graph_replay_ms(fn, reps):
    """Device time of each of `reps` replays of `fn` captured once into a CUDA graph."""
    g = B.GraphedCalls(fn)
    g()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def bench_chain64():
    """b2b_chain_vjp_f64 through 8 x PlanarLayer (Float64), D=128, N=2^16: x̄ and the w̄, ū, b̄ of every layer."""
    D, N, L = 128, 1 << 16, 8
    rng = np.random.default_rng(0)
    print_card()
    t = torch.float64
    flow = B.Composed(*[B.PlanarLayer(rng.standard_normal(D) / np.sqrt(D), rng.standard_normal(D) / np.sqrt(D),
                                      rng.standard_normal(1), dtype=t) for _ in range(L)])
    x = B.from_numpy(rng.standard_normal((D, N)), dtype=np.float64)
    yb = B.from_numpy(rng.standard_normal((D, N)), dtype=np.float64)
    lb = torch.from_numpy(rng.standard_normal(N)).cuda()
    ts = graph_replay_ms(lambda: B.chain_vjp(flow, x, yb, lb), 20)
    print(f"b2b_chain_vjp_f64 8 x Planar D={D} N=2^16: median {np.median(ts):.3f} ms, min {min(ts):.3f} ms (20 replays)")


def bench_chain():
    D, N, L = 128, 1 << 20, 8
    rng = np.random.default_rng(0)
    print_card()

    def device_ms(fn, reps=20):
        """Device time of one call: the call is captured once into a CUDA graph (no host work in the timed window) and
        the graph is replayed `reps` times between two events.  Every D x N operand is 512 MiB, far beyond the 50 MB L2,
        so back-to-back replays read from HBM."""
        g = B.GraphedCalls(fn)
        g()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    def report(name, t, nbytes):
        gbs = nbytes / t / 1e6
        print(f"{name}  D={D} N=2^20  {t:.4f} ms  {gbs:.0f} GB/s  ({gbs / 3350.0 * 100:.1f} % of the 3350 GB/s H100 data sheet)")

    # (a) the elementwise-run kernel: Stacked(Logit rows | exp rows) + Permute + MvNormal(μ, σ), ȳ = NULL, l̄ = 1 -- one
    # segment, so the call is the kernel plus the tiny fixed-order finalize of μ̄, σ̄
    st = B.Stacked([B.Logit(0.0, 1.0), B.elementwise("exp")], [(1, D // 2), (D // 2 + 1, D)])
    base = B.MvNormal(D, mu=(rng.standard_normal(D) * 0.1).astype(np.float32), sigma=rng.uniform(0.8, 1.2, D).astype(np.float32))
    td = B.transformed(base, B.inverse(B.Composed(st, B.Permute((rng.permutation(D) + 1).tolist()))))
    y = B.from_numpy(np.concatenate([rng.uniform(0.05, 0.95, (D // 2, N)), rng.standard_normal((D // 2, N))]).astype(np.float32))
    ones = torch.ones(N, device="cuda")
    report("(a) elementwise-run VJP kernel (Stacked + Permute + MvNormal, with μ̄, σ̄)", device_ms(lambda: B.logpdf_vjp(td, y, ones)),
           4.0 * N * (2 * D + 1))
    # (b) logpdf gradient of inverse(8 x Planar) + MvNormal: one chain_vjp call vs today's route, both as device time
    flow = B.Composed(*[B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                      (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                      rng.standard_normal(1).astype(np.float32)) for _ in range(L)])
    tdp = B.transformed(B.MvNormal(D), flow)
    yp = B.from_numpy(rng.standard_normal((D, N)).astype(np.float32))

    def today():
        x, _ = B.run_chain(B.inverse(flow), yp)  # the base density's cotangent is −x (torch)
        B.planar_chain_vjp(B.inverse(flow), yp, (-x).t().contiguous().t(), ones)

    ta, tb = [], []
    for _ in range(3):
        ta.append(device_ms(lambda: B.logpdf_vjp(tdp, yp, ones)))
        tb.append(device_ms(today))
    t_new, t_old = float(np.median(ta)), float(np.median(tb))
    report("(b) logpdf gradient, chain_vjp (ȳ + parameter cotangents)", t_new, 4.0 * N * (2 * D + 1))
    report("(b) logpdf gradient, planar_chain_vjp + torch base density", t_old, 4.0 * N * (2 * D + 1))
    print(f"(b) ratio today / chain_vjp: {t_old / t_new:.3f}  (per-run medians: chain_vjp {ta}, today {tb})")


if len(sys.argv) > 1 and sys.argv[1] == "chain":
    bench_chain()
    sys.exit(0)
if len(sys.argv) > 1 and sys.argv[1] == "chain64":
    bench_chain64()
    sys.exit(0)

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
