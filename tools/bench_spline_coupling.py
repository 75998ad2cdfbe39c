"""Times the spline coupling layer (B2B_COUPLING_RQS) as the device time of graph-captured calls (median of 20 replays,
three rounds), at D = 64 (n1 = n2 = 32), K = 8, N = 2^20 and D = 256 (n1 = n2 = 128), K = 8, N = 2^18:

  - the forward (b2b_chain_run_f32 on the one-layer chain, y and logjac written);
  - logpdf of transformed(MvNormal(D), layer): the inverse launch, then the fused MvNormal terminal;
  - the chain VJP of the inverse layer with x̄, W̄ and c̄ (b2b_chain_vjp_f32, l̄ = 1).

Each is reported against the larger of two bounds computed here from the shape: bytes over 3.35 TB/s (HBM3) and FP32 FMAs
over 67 TFLOP/s (33.5 T FMA/s), both H100 SXM data-sheet figures at 700 W.  Bytes: 4·(2D+1) B/sample (read x, write y and
logjac).  FMAs: (3K−1)·n1·n2 per sample for the conditioner GEMM of the forward and the inverse, 3× that for the VJP (the
GEMM recomputed, Wᵀr̄ and the W̄ outer product).  The bound leaves out the ~4K MUFU operations per transformed element of
the normaliser (exp, log1pexp, division) and the spline itself."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B  # noqa: E402

PEAK_GBS = 3350.0      # H100 SXM HBM3, data sheet
PEAK_TFMAS = 67.0 / 2  # H100 SXM FP32, data sheet: 67 TFLOP/s = 33.5 T FMA/s


def print_card():
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(f"card: {torch.cuda.get_device_name()}, power limit, max SM clock: {power}")


def bound_ms(bytes_per_sample, fma_per_sample, N):
    """(bound in ms, which side bounds it)."""
    tb = bytes_per_sample * N / (PEAK_GBS * 1e9) * 1e3
    tf = fma_per_sample * N / (PEAK_TFMAS * 1e12) * 1e3
    return (tf, "FMA") if tf >= tb else (tb, "HBM")


def replay_median_ms(fn, reps=20):
    g = B.GraphedCalls(fn)
    g()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def bench(D, n1, K, N):
    rng = np.random.default_rng(D)
    n2 = D - n1
    J = 3 * K - 1
    Bv = 3.0
    W = (rng.standard_normal((J * n1, n2)) * 0.5 / np.sqrt(n2)).astype(np.float32)
    c = (rng.standard_normal(J * n1) * 0.3).astype(np.float32)
    lay = B.Coupling(B.SplineConditioner(W, c, K=K, B=Bv), B.PartitionMask(D, range(1, n1 + 1), range(n1 + 1, D + 1)))
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
    Wb, cb = torch.empty(J * n1 * n2, device="cuda"), torch.empty(J * n1, device="cuda")
    ptrs = (ctypes.c_void_p * 4)(Wb.data_ptr(), cb.data_ptr())
    ws_b = lib.b2b_chain_vjp_workspace_bytes(inv, 1, D, N)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    stream = lambda: torch.cuda.current_stream().cuda_stream

    def forward():
        B._lib.check(lib.b2b_chain_run_f32(fwd, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0,
                                           stream()), "b2b_chain_run_f32")

    def vjp():
        B._lib.check(lib.b2b_chain_vjp_f32(inv, 1, x.data_ptr(), None, lb.data_ptr(), xb.data_ptr(),
                                           ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b, stream()),
                     "b2b_chain_vjp_f32")

    fma = J * n1 * n2
    cases = [
        ("forward", forward, bound_ms(4 * (2 * D + 1), fma, N)),
        ("logpdf (inverse)", lambda: B.logpdf(td, x), bound_ms(4 * (2 * D + 1), fma, N)),
        ("VJP (x̄, W̄, c̄)", vjp, bound_ms(4 * (2 * D + 1), 3 * fma, N)),
    ]
    times = {name: [] for name, _, _ in cases}
    for _ in range(3):
        for name, fn, _ in cases:
            times[name].append(replay_median_ms(fn))
    logn = int(np.log2(N))
    for name, _, (tb, side) in cases:
        t = float(np.median(times[name]))
        print(f"{name:18s} D={D:4d} n1={n1:3d} K={K:2d} N=2^{logn}  {t:8.3f} ms  bound {tb:6.3f} ms ({side})"
              f"  {tb / t * 100:5.1f} % of bound  rounds {['%.3f' % v for v in times[name]]}")
    del x, y, xb, ws
    torch.cuda.empty_cache()


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print_card()
    bench(64, 32, 8, 1 << 20)
    bench(256, 128, 8, 1 << 18)
