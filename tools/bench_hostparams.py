"""Times the 8 x PlanarLayer headline chain (D=128, N=2^20) with device-resident vs host-resident parameters."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import bijectors_jl_b200 as B

B.lib().b2b_set_kernel_variant(int(os.environ.get('B2B_VARIANT', '0')))
D, N, L = int(sys.argv[1]) if len(sys.argv) > 1 else 128, 1 << 20, int(sys.argv[2]) if len(sys.argv) > 2 else 8
rng = np.random.default_rng(0)
layers = [B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                        (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                        rng.standard_normal(1).astype(np.float32)) for _ in range(L)]
dev, host = B.Composed(*layers), B.Composed(*[l.to("cpu") for l in layers])
x = B.from_numpy(rng.standard_normal((D, N)).astype(np.float32))
y, lj = B.colmajor_empty(D, N, "cuda"), torch.empty(N, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for name, flow in (("device", dev), ("host", host), ("device-inv", B.inverse(dev)), ("host-inv", B.inverse(host))):
    ts = []
    for it in range(13):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        B.run_chain(flow, x, y=y, logjac=lj)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    t = float(np.median(ts[3:]))
    gb = 4.0 * (2 * D + 1) * N / 1e9
    print(f"{name:11s} D={D} L={L}  {t:.4f} ms  {N / t / 1e6:.2f} G samples/s  {gb / t * 1e3:.0f} GB/s  ({gb / t * 1e3 / 3350.0 * 100:.1f} % of the 3350 GB/s H100 data sheet)")
