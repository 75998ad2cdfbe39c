"""Times the full-covariance MvNormal base (B2B_MVNORMAL_TRIL) at D = 128, 256 and N = 2^20, as the device time of
graph-captured calls (median of 20 replays, three rounds):

  - the TRIL logpdf launch alone (b2b_chain_run_f32 on the one-element chain, y = NULL);
  - logpdf of transformed(MvNormal(μ, L Lᵀ), 8×Planar) (the fused inverse planar chain, then the TRIL launch);
  - the chain VJP of the TRIL terminal with μ̄ and L̄ (b2b_chain_vjp_f32 on the one-element chain; the planar VJP kernels
    stop at D = 128, so the 8×Planar chain is not differentiated here);
  - rand of the base (b2b_chain_sample_tril_f32, L = 0 layers).

Each is reported against the larger of two bounds computed here from the shape: bytes over 3.35 TB/s (HBM3) and FP32 FMAs
over 67 TFLOP/s (33.5 T FMA/s), both H100 SXM data-sheet figures at 700 W.  Bytes: 4·(D+1) B/sample for the logpdf launch
(read x, write logpdf), 4·D for rand (the store).  FMAs: D(D+1)/2 per sample for the logpdf launch and for rand (the
triangular solve / product), 1.5·D(D+1) for the VJP (forward solve, back solve, and the L̄ outer product).  The 8×Planar
logpdf also moves the chain's own traffic, which the bound leaves out."""
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


def bench(D, N):
    rng = np.random.default_rng(D)
    L = np.tril(rng.standard_normal((D, D))) * (0.5 / np.sqrt(D))
    L[np.arange(D), np.arange(D)] = rng.uniform(0.7, 1.3, D)
    mu = (rng.standard_normal(D) * 0.3).astype(np.float32)
    base = B.MvNormal(D, mu=mu, scale_tril=L.astype(np.float32))
    flow = B.Composed(*[B.PlanarLayer((rng.standard_normal(D) * 0.1).astype(np.float32),
                                      (rng.standard_normal(D) * 0.1).astype(np.float32),
                                      rng.standard_normal(1).astype(np.float32)) for _ in range(8)])
    td = B.transformed(base, flow)
    y = B.colmajor_empty(D, N)
    y.copy_(torch.randn((N, D), device="cuda").t())
    lb = torch.ones(N, device="cuda")
    lib = B.lib()
    arr = (B._lib.LayerDesc * 1)(base._terminal_desc())
    lp = torch.empty(N, device="cuda")
    xb = B.colmajor_empty(D, N)
    mub, Lb = torch.empty(D, device="cuda"), torch.empty(D * D, device="cuda")
    ptrs = (ctypes.c_void_p * 4)(mub.data_ptr(), Lb.data_ptr())
    ws_b = lib.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    stream = lambda: torch.cuda.current_stream().cuda_stream

    def tril_launch():
        B._lib.check(lib.b2b_chain_run_f32(arr, 1, y.data_ptr(), None, lp.data_ptr(), None, D, N, D, D, 0, None, 0, stream()),
                     "b2b_chain_run_f32")

    def tril_vjp():
        B._lib.check(lib.b2b_chain_vjp_f32(arr, 1, y.data_ptr(), None, lb.data_ptr(), xb.data_ptr(),
                                           ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b, stream()),
                     "b2b_chain_vjp_f32")

    cases = [
        ("TRIL logpdf launch", tril_launch, bound_ms(4 * (D + 1), D * (D + 1) / 2, N)),
        ("logpdf 8xPlanar+TRIL", lambda: B.logpdf(td, y), bound_ms(4 * (D + 1), D * (D + 1) / 2, N)),
        ("TRIL VJP (x̄, μ̄, L̄)", tril_vjp, bound_ms(4 * (2 * D + 1), 1.5 * D * (D + 1), N)),
        ("rand", lambda: base.rand(N, seed=1), bound_ms(4 * D, D * (D + 1) / 2, N)),
    ]
    times = {name: [] for name, _, _ in cases}
    for _ in range(3):
        for name, fn, _ in cases:
            times[name].append(replay_median_ms(fn))
    logn = int(np.log2(N))
    for name, _, (tb, side) in cases:
        t = float(np.median(times[name]))
        print(f"{name:22s} D={D:4d} N=2^{logn}  {t:8.3f} ms  bound {tb:6.3f} ms ({side})  {tb / t * 100:5.1f} % of bound"
              f"  rounds {['%.3f' % v for v in times[name]]}")
    del y
    torch.cuda.empty_cache()


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print_card()
    for D in (128, 256):
        bench(D, 1 << 20)
