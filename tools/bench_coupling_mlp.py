"""Times the neural-network coupling layer (B2B_COUPLING_MLP, tanh) as the device time of graph-captured calls (median of
20 replays, three rounds) at N = 2^20: D = 64 (n1 = n2 = 32, H = 64) and D = 256 (n1 = n2 = 128) with H = 128 and H = 256:

  - the forward and the inverse (b2b_chain_run_f32 on the one-layer chain, y and logjac written);
  - logpdf of transformed(MvNormal(D), layer): the inverse launch, then the fused MvNormal terminal;
  - the chain VJP of the inverse layer with x̄, W̄₁, c̄₁, W̄₂, c̄₂ (b2b_chain_vjp_f32, l̄ = 1);

and, alternated with them in the same rounds, the linear COUPLING_AFFINE layer of the same mask on the exact-fp32
CUDA-core kernel (kernel variant 10).

Each is reported against the larger of two bounds computed here from the shape: bytes over 3.35 TB/s (HBM3) and FP32 FMAs
over 67 TFLOP/s (33.5 T FMA/s), both H100 SXM data-sheet figures at 700 W.  Bytes: 4·(2D+1) B/sample (read x, write y and
logjac).  FMAs per sample: H·(n2 + 2·n1) for the network (2·n1·n2 for the affine layer), 3× that for the VJP (the
network recomputed, the two transposed products, the two outer products)."""
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


def bench(D, n1, H, N):
    rng = np.random.default_rng(D + H)
    n2 = D - n1
    mask = B.PartitionMask(D, range(1, n1 + 1), range(n1 + 1, D + 1))
    W1 = (rng.standard_normal((H, n2)) * 0.5 / np.sqrt(n2)).astype(np.float32)
    W2 = (rng.standard_normal((2 * n1, H)) * 0.5 / np.sqrt(H)).astype(np.float32)
    c1, c2 = (rng.standard_normal(H) * 0.3).astype(np.float32), (rng.standard_normal(2 * n1) * 0.3).astype(np.float32)
    mlp = B.Coupling(B.MLPConditioner(W1, c1, W2, c2), mask)
    aff = B.Coupling(B.AffineConditioner((rng.standard_normal((2 * n1, n2)) * 0.5 / np.sqrt(n2)).astype(np.float32), c2), mask)
    x = B.colmajor_empty(D, N)
    x.copy_(torch.randn((N, D), device="cuda").t())
    y = B.colmajor_empty(D, N)
    lj = torch.empty(N, device="cuda")
    lb = torch.ones(N, device="cuda")
    xb = B.colmajor_empty(D, N)
    lib = B.lib()
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    B._lib.check(lib.b2b_set_kernel_variant(10), "b2b_set_kernel_variant")  # the affine layer on the exact-fp32 kernel
    cases = []
    for name, lay, fma, nslots in (("MLP", mlp, H * (n2 + 2 * n1), 4), ("affine", aff, 2 * n1 * n2, 2)):
        fwd = (B._lib.LayerDesc * 1)(*lay._descs(False, D))
        inv = (B._lib.LayerDesc * 1)(*lay._descs(True, D))
        bars = [torch.empty(2 * n1 * max(H, n2) + H * n2, device="cuda") for _ in range(nslots)]
        ptrs = (ctypes.c_void_p * 4)(*[b.data_ptr() for b in bars])
        ws_b = lib.b2b_chain_vjp_workspace_bytes(inv, 1, D, N)
        ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
        td = B.transformed(B.MvNormal(D), lay)

        def run(arr=fwd):
            B._lib.check(lib.b2b_chain_run_f32(arr, 1, x.data_ptr(), y.data_ptr(), lj.data_ptr(), None, D, N, D, D, 0, None, 0,
                                               stream()), "b2b_chain_run_f32")

        def vjp(inv=inv, ptrs=ptrs, ws=ws, ws_b=ws_b):
            B._lib.check(lib.b2b_chain_vjp_f32(inv, 1, x.data_ptr(), None, lb.data_ptr(), xb.data_ptr(),
                                               ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b, stream()),
                         "b2b_chain_vjp_f32")

        byt = 4 * (2 * D + 1)
        cases += [(f"{name} forward", run, bound_ms(byt, fma, N)),
                  (f"{name} inverse", lambda inv=inv, run=run: run(inv), bound_ms(byt, fma, N)),
                  (f"{name} logpdf", lambda td=td: B.logpdf(td, x), bound_ms(byt, fma, N)),
                  (f"{name} VJP (all cotangents)", vjp, bound_ms(byt, 3 * fma, N))]
    times = {name: [] for name, _, _ in cases}
    for _ in range(3):
        for k in range(4):  # MLP and affine alternate
            for name, fn, _ in (cases[k], cases[4 + k]):
                times[name].append(replay_median_ms(fn))
    logn = int(np.log2(N))
    for k in range(4):
        for name, _, (tb, side) in (cases[k], cases[4 + k]):
            t = float(np.median(times[name]))
            print(f"{name:28s} D={D:4d} n1={n1:3d} H={H:3d} N=2^{logn}  {t:8.3f} ms  bound {tb:6.3f} ms ({side})"
                  f"  {tb / t * 100:5.1f} % of bound  rounds {['%.3f' % v for v in times[name]]}")
    B._lib.check(lib.b2b_set_kernel_variant(0), "b2b_set_kernel_variant")
    del x, y, xb, cases
    torch.cuda.empty_cache()


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print_card()
    bench(64, 32, 64, 1 << 20)
    bench(256, 128, 128, 1 << 20)
    bench(256, 128, 256, 1 << 20)
