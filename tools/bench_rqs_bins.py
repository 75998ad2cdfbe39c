"""Spline layer, D = 32, N = 2^19: the specialised program (auto) against the layer interpreter (kernel variant 2) for bin
counts with and without a table of their own (K = 8, 16 have one; K = 6, 10, 20 run in the next larger table)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B

D, N = 32, 1 << 19
rng = np.random.default_rng(0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
x = B.from_numpy((rng.standard_normal((D, N)) * 1.5).astype(np.float32))


def timed(fn, reps=15):
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts[3:]))


for K in (8, 6, 10, 16, 20):
    sp = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(np.float32), rng.standard_normal((D, K)).astype(np.float32),
                                   rng.standard_normal((D, K - 1)).astype(np.float32), 3.0)
    row = []
    for variant in (0, 2):
        B.lib().b2b_set_kernel_variant(variant)
        try:
            row.append((timed(lambda: B.with_logabsdet_jacobian(sp, x)), timed(lambda: B.with_logabsdet_jacobian(B.inverse(sp), x))))
        finally:
            B.lib().b2b_set_kernel_variant(0)
    gb = 4.0 * N * (2 * D + 1) / 1e9
    print(f"K={K:2d}  program fwd {row[0][0]*1e3:6.1f} us ({gb/row[0][0]*1e3/3350.0*100:4.1f} %)  inv {row[0][1]*1e3:6.1f} us ({gb/row[0][1]*1e3/3350.0*100:4.1f} %)"
          f"   interpreter fwd {row[1][0]*1e3:6.1f} us  inv {row[1][1]*1e3:6.1f} us")
