"""Times the deep neural spline coupling layer (B2B_COUPLING_DEEP_MLP_RQS) at M = 2, 3, 4 hidden layers as the device
time of graph-captured calls (median of 20 replays, three rounds), alternated in the same call with the one-hidden-layer
neural spline coupling (B2B_COUPLING_MLP_RQS) at the same n1, n2, H and K: D = 64 (n1 = n2 = 32, H = 64), N = 2^20 and
D = 256 (n1 = n2 = H = 128), N = 2^18, both at K = 8 -- the shapes of tools/bench_coupling_mlp_rqs.py.

The three runs of each layer are those of tools/bench_coupling_mlp_rqs.py: the forward, logpdf of
transformed(MvNormal(D), layer), and the chain VJP of the inverse layer with x̄ and all four parameter cotangents.  The
FP32-FMA bound counts H·n2 + (M − 1)·H² + (3K − 1)·n1·H FMAs per sample for the forward and the inverse, 3× that for the
VJP; the last column is the time over kind 14's, next to the FMA ratio."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bijectors_jl_b200 as B  # noqa: E402
from bench_coupling_mlp_rqs import cases  # noqa: E402
from bench_spline_coupling import print_card, replay_median_ms  # noqa: E402


def bench(D, n1, H, K, N):
    rng = np.random.default_rng(D)
    n2 = D - n1
    J = (3 * K - 1) * n1
    Bv = 3.0
    mask = B.PartitionMask(D, range(1, n1 + 1), range(n1 + 1, D + 1))
    W_in = (rng.standard_normal((H, n2)) / np.sqrt(n2)).astype(np.float32)
    W_out = (rng.standard_normal((J, H)) * 0.5 / np.sqrt(H)).astype(np.float32)
    c = [(rng.standard_normal(H) * 0.3).astype(np.float32) for _ in range(4)]
    c_out = (rng.standard_normal(J) * 0.3).astype(np.float32)
    hid = [(rng.standard_normal((H, H)) / np.sqrt(H)).astype(np.float32) for _ in range(3)]
    fma14 = H * n2 + J * H
    runs = cases("M=1 (kind 14)", B.Coupling(B.MLPSplineConditioner(W_in, c[0], W_out, c_out, K=K, B=Bv), mask), D,
                 fma14, N)
    fma = {1: fma14}
    for M in (2, 3, 4):
        cond = B.DeepMLPSplineConditioner([W_in] + hid[:M - 1] + [W_out], c[:M] + [c_out], K=K, B=Bv)
        fma[M] = fma14 + (M - 1) * H * H
        runs += cases(f"M={M}", B.Coupling(cond, mask), D, fma[M], N)
    times = {name: [] for name, _, _, _ in runs}
    for _ in range(3):
        for name, fn, _, _ in runs:
            times[name].append(replay_median_ms(fn))
    logn = int(np.log2(N))
    med = {name: float(np.median(v)) for name, v in times.items()}
    for name, _, (tb, side), _ in runs:
        t = med[name]
        M = int(name.split("=")[1][0])
        what = name.split()[-1]
        base = med[f"M=1 (kind 14) {what}"]
        print(f"{name:22s} D={D:4d} n1={n1:3d} H={H:3d} K={K:2d} N=2^{logn}  {t:8.3f} ms  bound {tb:6.3f} ms ({side})"
              f"  {tb / t * 100:5.1f} % of bound  {t / base:5.3f}x kind 14 (FMA {fma[M] / fma14:4.2f}x)"
              f"  rounds {['%.3f' % v for v in times[name]]}")
    del runs
    torch.cuda.empty_cache()


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print_card()
    bench(64, 32, 64, 8, 1 << 20)
    bench(256, 128, 128, 8, 1 << 18)
