"""Times the dense Scale layer (B2B_SCALE_MATRIX) at D = 64, 128, 256 and N = 2^20 as the device time of graph-captured
calls (median of 20 replays, three rounds), prints the card and its power limit, and writes the table to --out
(default records/bench_scale_matrix_h100.txt):

  - forward  y = A x          (factor launch, then the map GEMM)
  - inverse  y = A⁻¹ x        (factor, A⁻¹ solves, map GEMM)
  - logpdf of transformed(MvNormal(μ, Diagonal(σ²)), Scale(A))   (the inverse layer, then the fused diagonal terminal)
  - VJP of the forward layer with x̄ and Ā (ȳ and l̄ given)
  - the factor alone: the forward and the inverse call at N = 1

Each call is reported against the larger of two bounds computed from the shape with H100 SXM data-sheet figures: D²·N FP32
FMAs (2·D²·N for the VJP: the transposed map and the G = Σ ȳ uᵀ product) over 33.5 T FMA/s, and (8D + 4)·N bytes (read x,
write y and the log-Jacobian; the VJP reads u and ȳ and writes x̄, (12D + 4)·N) over 3.35 TB/s."""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bijectors_jl_b200 as B  # noqa: E402

PEAK_GBS = 3350.0      # H100 SXM HBM3, data sheet
PEAK_TFMAS = 67.0 / 2  # H100 SXM FP32, data sheet: 67 TFLOP/s = 33.5 T FMA/s


def card():
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return f"card: {torch.cuda.get_device_name()}, power limit, max SM clock: {power}"


def bound_ms(bytes_per_sample, fma_per_sample, N):
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


def bench(D, N, lines):
    rng = np.random.default_rng(D)
    A = (np.eye(D) + 0.3 * rng.standard_normal((D, D)) / np.sqrt(D)).astype(np.float32)
    lay = B.Scale(A)
    inv = B.inverse(lay)
    base = B.MvNormal(D, mu=(rng.standard_normal(D) * 0.3).astype(np.float32), sigma=rng.uniform(0.7, 1.3, D).astype(np.float32))
    td = B.transformed(base, lay)
    x = B.colmajor_empty(D, N)
    x.copy_(torch.randn((N, D), device="cuda").t())
    y = B.colmajor_empty(D, N)
    lj = torch.empty(N, device="cuda")
    yb = B.colmajor_empty(D, N)
    yb.copy_(torch.randn((N, D), device="cuda").t())
    lb = torch.ones(N, device="cuda")
    x1, y1, lj1 = B.colmajor_empty(D, 1), B.colmajor_empty(D, 1), torch.empty(1, device="cuda")
    x1.zero_()
    lib = B.lib()
    arr = (B._lib.LayerDesc * 1)(*lay._descs(False, D))
    xbar = B.colmajor_empty(D, N)
    abar = torch.empty(D * D, device="cuda")
    ptrs = (ctypes.c_void_p * 4)(abar.data_ptr())
    ws_b = lib.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731

    def vjp():
        B._lib.check(lib.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), yb.data_ptr(), lb.data_ptr(), xbar.data_ptr(),
                                           ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b, stream()),
                     "b2b_chain_vjp_f32")

    cases = [
        ("forward", lambda: B.run_chain(lay, x, y=y, logjac=lj), bound_ms(8 * D + 4, D * D, N)),
        ("inverse", lambda: B.run_chain(inv, x, y=y, logjac=lj), bound_ms(8 * D + 4, D * D, N)),
        ("logpdf (diagonal base)", lambda: B.logpdf(td, x), bound_ms(8 * D + 4, D * D, N)),
        ("VJP (x̄, Ā)", vjp, bound_ms(12 * D + 4, 2 * D * D, N)),
        ("factor: forward, N = 1", lambda: B.run_chain(lay, x1, y=y1, logjac=lj1), None),
        ("factor: inverse, N = 1", lambda: B.run_chain(inv, x1, y=y1, logjac=lj1), None),
    ]
    times = {name: [] for name, _, _ in cases}
    for _ in range(3):
        for name, fn, _ in cases:
            times[name].append(replay_median_ms(fn))
    logn = int(np.log2(N))
    for name, _, bnd in cases:
        t = float(np.median(times[name]))
        rounds = ["%.3f" % v for v in times[name]]
        if bnd is None:
            line = f"{name:24s} D={D:4d}          {t:8.3f} ms  rounds {rounds}"
        else:
            tb, side = bnd
            line = (f"{name:24s} D={D:4d} N=2^{logn}  {t:8.3f} ms  bound {tb:6.3f} ms ({side})  {tb / t * 100:5.1f} % of bound"
                    f"  rounds {rounds}")
        print(line, flush=True)
        lines.append(line)
    del x, y, yb, xbar
    torch.cuda.empty_cache()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "bench_scale_matrix_h100.txt"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    lines = [card()]
    print(lines[0], flush=True)
    for D in (64, 128, 256):
        bench(D, 1 << 20, lines)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
