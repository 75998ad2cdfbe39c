"""Times b2b_batchnorm_train_vjp_f32 (reverse mode of the training-mode InvertibleBatchNorm) at D = 64, 256 (N = 2^22) and
D = 1024 (N = 2^20), as the device time of graph-captured calls (median of 20 replays), against b2b_batchnorm_eval_vjp_f32
at the same shape -- the column-local reverse mode, which reads x and ȳ once.  The two are alternated, three rounds each.
Bytes are the algorithmic traffic: 4·(5D + 1) per column for the training-mode call (pass 1 reads x, ȳ, l̄; pass 2 reads
x, ȳ and writes x̄), 4·(3D + 1) for the eval-mode one.  Every D x N operand is at least 1 GiB, far beyond the 50 MB L2,
so back-to-back replays read from HBM."""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B  # noqa: E402
from bijectors_jl_b200._lib import LayerDesc  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet


def print_card():
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(f"card: {torch.cuda.get_device_name()}, power limit: {power}")


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
    L_ = B._lib.lib()
    gen = torch.Generator(device="cuda").manual_seed(D)
    x = (torch.randn((N, D), device="cuda", generator=gen) * 1.7 + 0.3).t()
    yb = torch.randn((N, D), device="cuda", generator=gen).t()
    lb = torch.randn(N, device="cuda", generator=gen)
    xb = B.colmajor_empty(D, N)
    bbar, lbar = torch.empty(D, device="cuda"), torch.empty(D, device="cuda")
    bn = B.InvertibleBatchNorm(b=np.zeros(D, np.float32), logs=np.full(D, 0.1, np.float32), m=np.zeros(D, np.float32),
                               v=np.ones(D, np.float32))
    ws_t = L_.b2b_batchnorm_train_vjp_workspace_bytes(D)
    ws_e = L_.b2b_batchnorm_eval_vjp_workspace_bytes(D)
    ws = torch.empty((max(ws_t, ws_e),), dtype=torch.uint8, device="cuda")
    desc = (LayerDesc * 1)(*bn._descs(False, D))
    stream = lambda: torch.cuda.current_stream().cuda_stream

    def train():
        B._lib.check(L_.b2b_batchnorm_train_vjp_f32(x.data_ptr(), yb.data_ptr(), lb.data_ptr(), xb.data_ptr(), bbar.data_ptr(),
                                                    lbar.data_ptr(), bn.logs.data_ptr(), bn.eps, D, N, D, D, D, None,
                                                    ws.data_ptr(), ws_t, stream()), "b2b_batchnorm_train_vjp_f32")

    def evalm():
        B._lib.check(L_.b2b_batchnorm_eval_vjp_f32(desc, x.data_ptr(), yb.data_ptr(), lb.data_ptr(), xb.data_ptr(),
                                                   bbar.data_ptr(), lbar.data_ptr(), D, N, D, D, D, ws.data_ptr(), ws_e,
                                                   stream()), "b2b_batchnorm_eval_vjp_f32")

    tt, te = [], []
    for _ in range(3):
        tt.append(replay_median_ms(train))
        te.append(replay_median_ms(evalm))
    logn = int(np.log2(N))
    for name, ts, per_col in (("train-mode VJP", tt, 5 * D + 1), ("eval-mode VJP ", te, 3 * D + 1)):
        t = float(np.median(ts))
        gbs = 4.0 * per_col * N / t / 1e6
        print(f"{name} D={D:5d} N=2^{logn}  {t:8.3f} ms  {gbs:6.0f} GB/s  ({gbs / PEAK_GBS * 100:5.1f} % of {PEAK_GBS:.0f} GB/s)"
              f"  rounds {['%.3f' % v for v in ts]}")
    del x, yb, xb
    torch.cuda.empty_cache()


if __name__ == "__main__":
    torch.cuda.set_device(0)
    print_card()
    for D, N in ((64, 1 << 22), (256, 1 << 22), (1024, 1 << 20)):
        bench(D, N)
