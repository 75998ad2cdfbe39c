"""Times the deep neural-network coupling layer (B2B_COUPLING_DEEP_MLP, tanh) as the device time of graph-captured calls
(median of 20 replays, three rounds) at D = 256, N = 2^20, n1 = n2 = H = 128, with M = 2, 3 and 4 hidden layers:

  - the forward and the inverse (b2b_chain_run_f32 on the one-layer chain, y and logjac written);
  - the chain VJP of the inverse layer with x̄, W̄_in, W̄_hid, W̄_out, c̄ (b2b_chain_vjp_f32, l̄ = 1);

and, alternated with them in the same rounds, the one-hidden-layer B2B_COUPLING_MLP of the same mask and H.

Each is reported against the larger of two bounds computed here from the shape: bytes over 3.35 TB/s (HBM3) and FP32 FMAs
over 67 TFLOP/s (33.5 T FMA/s), both H100 SXM data-sheet figures at 700 W.  Bytes: 4·(2D+1) B/sample (read x, write y and
logjac).  FMAs per sample: H·n2 + (M−1)·H² + 2·n1·H for the forward network (2·(…) FLOP), 3× that for the VJP (the
network recomputed, the transposed products, the outer products)."""
import ctypes
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bijectors_jl_b200 as B  # noqa: E402
from bench_coupling_mlp import bound_ms, print_card, replay_median_ms  # noqa: E402


def bench(D, n1, H, N, depths=(2, 3, 4)):
    rng = np.random.default_rng(D + H)
    n2 = D - n1
    mask = B.PartitionMask(D, range(1, n1 + 1), range(n1 + 1, D + 1))
    W_in = (rng.standard_normal((H, n2)) * 0.5 / np.sqrt(n2)).astype(np.float32)
    W_out = (rng.standard_normal((2 * n1, H)) * 0.5 / np.sqrt(H)).astype(np.float32)
    c = [(rng.standard_normal(H) * 0.3).astype(np.float32) for _ in range(max(depths))]
    c_out = (rng.standard_normal(2 * n1) * 0.3).astype(np.float32)
    W_hid = [(rng.standard_normal((H, H)) * 1.0 / np.sqrt(H)).astype(np.float32) for _ in range(max(depths) - 1)]
    layers = [("MLP (M = 1)", B.Coupling(B.MLPConditioner(W_in, c[0], W_out, c_out), mask), 1)]
    for M in depths:
        cond = B.DeepMLPConditioner([W_in] + W_hid[:M - 1] + [W_out], c[:M] + [c_out])
        layers.append((f"deep MLP (M = {M})", B.Coupling(cond, mask), M))
    x = B.colmajor_empty(D, N)
    x.copy_(torch.randn((N, D), device="cuda").t())
    y = B.colmajor_empty(D, N)
    lj = torch.empty(N, device="cuda")
    lb = torch.ones(N, device="cuda")
    xb = B.colmajor_empty(D, N)
    lib = B.lib()
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    byt = 4 * (2 * D + 1)
    groups = []
    for name, lay, M in layers:
        fwd = (B._lib.LayerDesc * 1)(*lay._descs(False, D))
        inv = (B._lib.LayerDesc * 1)(*lay._descs(True, D))
        bars = [torch.empty(max(M - 1, 1) * H * H + 2 * n1 * H + H * n2, device="cuda") for _ in range(4)]
        ptrs = (ctypes.c_void_p * 4)(*[b.data_ptr() for b in bars])
        ws_b = lib.b2b_chain_vjp_workspace_bytes(inv, 1, D, N)
        ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
        fma = H * n2 + (M - 1) * H * H + 2 * n1 * H

        def run(arr=fwd):
            B._lib.check(lib.b2b_chain_run_f32(arr, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0,
                                               stream()), "b2b_chain_run_f32")

        def vjp(inv=inv, ptrs=ptrs, ws=ws, ws_b=ws_b, bars=bars):
            B._lib.check(lib.b2b_chain_vjp_f32(inv, 1, x.data_ptr(), None, lb.data_ptr(), xb.data_ptr(),
                                               ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b, stream()),
                         "b2b_chain_vjp_f32")

        groups.append([(f"{name} forward", run, bound_ms(byt, fma, N)),
                       (f"{name} inverse", lambda inv=inv, run=run: run(inv), bound_ms(byt, fma, N)),
                       (f"{name} VJP (all cotangents)", vjp, bound_ms(byt, 3 * fma, N))])
    times = {name: [] for grp in groups for name, _, _ in grp}
    for _ in range(3):
        for k in range(3):  # the layers alternate call by call
            for grp in groups:
                name, fn, _ = grp[k]
                times[name].append(replay_median_ms(fn))
    logn = int(np.log2(N))
    base = {k: float(np.median(times[groups[0][k][0]])) for k in range(3)}
    for k in range(3):
        for grp in groups:
            name, _, (tb, side) = grp[k]
            t = float(np.median(times[name]))
            print(f"{name:40s} D={D:4d} n1={n1:3d} H={H:3d} N=2^{logn}  {t:8.3f} ms  {t / base[k]:5.2f}x M = 1  "
                  f"bound {tb:6.3f} ms ({side})  {tb / t * 100:5.1f} % of bound  rounds {['%.3f' % v for v in times[name]]}")
    del x, y, xb, groups
    torch.cuda.empty_cache()


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print_card()
    bench(256, 128, 128, 1 << 20)
