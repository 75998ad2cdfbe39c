"""Times rand(td, n): base samples generated inside the chain kernel (b2b_chain_sample_f32) vs. base samples written to HBM
and pushed through the chain in a second pass, for the headline chain (8 x PlanarLayer, D=128, N=2^20)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B

D, N, L = 128, 1 << 20, 8
rng = np.random.default_rng(0)
flow = B.Composed(*[B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                  (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                  rng.standard_normal(1).astype(np.float32)) for _ in range(L)])
base = B.MvNormal(D)
td = B.transformed(base, flow)
peak = 3350.0  # GB/s, H100 SXM data-sheet HBM3 bandwidth


def timed(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


ms = timed(lambda: B.rand(td, N, seed=1))
print(f"fused sampler (Philox in the chain kernel): {ms:.4f} ms  {N / ms / 1e6:.2f} G samples/s  "
      f"{4 * (D) * N / ms / 1e6 / peak:.3f} of the 4*D B/sample store roofline")
ms0 = timed(lambda: base.rand(N, seed=1))
print(f"base samples only (b2b_randn_f32):          {ms0:.4f} ms  {N / ms0 / 1e6:.2f} G samples/s")
z = base.rand(N, seed=1)
y = B.colmajor_empty(D, N)
ms1 = timed(lambda: B.run_chain(flow, z, y=y, want_logjac=False))
print(f"two passes (randn, then the chain):          {ms0 + ms1:.4f} ms")
ms2 = timed(lambda: torch.randn((N, D), device="cuda"))
print(f"torch.randn of the same shape:               {ms2:.4f} ms")
