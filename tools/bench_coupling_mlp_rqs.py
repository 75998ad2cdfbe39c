"""Times the neural spline coupling layer (B2B_COUPLING_MLP_RQS) as the device time of graph-captured calls (median of 20
replays, three rounds), at D = 64 (n1 = n2 = 32, H = 64), K = 8, N = 2^20 and D = 256 (n1 = n2 = H = 128), K = 8,
N = 2^18:

  - the forward (b2b_chain_run_f32 on the one-layer chain, y and logjac written);
  - logpdf of transformed(MvNormal(D), layer): the inverse launch, then the fused MvNormal terminal;
  - the chain VJP of the inverse layer with x̄ and all four parameter cotangents (b2b_chain_vjp_f32, l̄ = 1).

Each is reported against its FP32-FMA bound as in tools/bench_spline_coupling.py: H·n2 + (3K−1)·n1·H FMAs per sample for
the forward and the inverse, 3× that for the VJP.  Next to it, in the same call, the same three runs of the linear spline
coupling (B2B_COUPLING_RQS) with n2 := H conditioning rows (a batch of n1 + H rows), whose conditioner GEMM is the new
layer's dominant one: the network adds the H·n2 FMAs of its hidden layer."""
import ctypes
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bijectors_jl_b200 as B  # noqa: E402
from bench_spline_coupling import bound_ms, print_card, replay_median_ms  # noqa: E402


def cases(name, lay, D, fma, N):
    """The three timed runs of the one-layer chain `lay` at D."""
    td = B.transformed(B.MvNormal(D), lay)
    x = B.colmajor_empty(D, N)
    x.copy_(torch.randn((N, D), device="cuda").t())
    y = B.colmajor_empty(D, N)
    lj = torch.empty(N, device="cuda")
    lib = B.lib()
    fwd = (B._lib.LayerDesc * 1)(*lay._descs(False, D))
    inv = (B._lib.LayerDesc * 1)(*lay._descs(True, D))
    lb = torch.ones(N, device="cuda")
    xb = B.colmajor_empty(D, N)
    from bijectors_jl_b200.interface import _slot_shape

    bars = [torch.empty(_slot_shape(inv[0], i, D), device="cuda") if p else None
            for i, p in enumerate((inv[0].p0, inv[0].p1, inv[0].p2, inv[0].p3))]
    ptrs = (ctypes.c_void_p * 4)(*[None if b is None else b.data_ptr() for b in bars])
    ws_b = lib.b2b_chain_vjp_workspace_bytes(inv, 1, D, N)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731

    def forward():
        B._lib.check(lib.b2b_chain_run_f32(fwd, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0,
                                           stream()), "b2b_chain_run_f32")

    def vjp():
        B._lib.check(lib.b2b_chain_vjp_f32(inv, 1, x.data_ptr(), None, lb.data_ptr(), xb.data_ptr(),
                                           ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b, stream()),
                     "b2b_chain_vjp_f32")

    keep = (x, y, lj, lb, xb, bars, ws)
    return [(f"{name} forward", forward, bound_ms(4 * (2 * D + 1), fma, N), keep),
            (f"{name} logpdf", lambda: B.logpdf(td, x), bound_ms(4 * (2 * D + 1), fma, N), keep),
            (f"{name} VJP", vjp, bound_ms(4 * (2 * D + 1), 3 * fma, N), keep)]


def bench(D, n1, H, K, N):
    rng = np.random.default_rng(D)
    n2 = D - n1
    J = 3 * K - 1
    Bv = 3.0
    W1 = (rng.standard_normal((H, n2)) / np.sqrt(n2)).astype(np.float32)
    c1 = (rng.standard_normal(H) * 0.3).astype(np.float32)
    W2 = (rng.standard_normal((J * n1, H)) * 0.5 / np.sqrt(H)).astype(np.float32)
    c2 = (rng.standard_normal(J * n1) * 0.3).astype(np.float32)
    nsf = B.Coupling(B.MLPSplineConditioner(W1, c1, W2, c2, K=K, B=Bv),
                     B.PartitionMask(D, range(1, n1 + 1), range(n1 + 1, D + 1)))
    Dl = n1 + H  # the linear spline coupling conditioned on H rows
    lin = B.Coupling(B.SplineConditioner(W2, c2, K=K, B=Bv), B.PartitionMask(Dl, range(1, n1 + 1), range(n1 + 1, Dl + 1)))
    runs = cases("MLP_RQS", nsf, D, H * n2 + J * n1 * H, N) + cases(f"RQS n2={H}", lin, Dl, J * n1 * H, N)
    times = {name: [] for name, _, _, _ in runs}
    for _ in range(3):
        for name, fn, _, _ in runs:
            times[name].append(replay_median_ms(fn))
    logn = int(np.log2(N))
    med = {name: float(np.median(v)) for name, v in times.items()}
    for name, _, (tb, side), _ in runs:
        t = med[name]
        print(f"{name:18s} D={D:4d} n1={n1:3d} H={H:3d} K={K:2d} N=2^{logn}  {t:8.3f} ms  bound {tb:6.3f} ms ({side})"
              f"  {tb / t * 100:5.1f} % of bound  rounds {['%.3f' % v for v in times[name]]}")
    for what in ("forward", "logpdf", "VJP"):
        print(f"  MLP_RQS / RQS (n2 = H) {what}: {med['MLP_RQS ' + what] / med[f'RQS n2={H} ' + what]:.3f}x")
    del runs
    torch.cuda.empty_cache()


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print_card()
    bench(64, 32, 64, 8, 1 << 20)
    bench(256, 128, 128, 8, 1 << 18)
