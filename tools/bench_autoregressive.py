"""Times the masked autoregressive layer (B2B_AUTOREGRESSIVE_MLP, MaskedAutoregressive) at N = 2^20, D in {16, 64, 128}
and H in {64, 256} with the method of tools/bench_scale_matrix.py (device time of graph-captured calls, median of the
replays, three rounds; the card and its power limit read in the same run), and writes the table to --out (default
records/bench_autoregressive_h100.txt).  Calls, each with its prep launch:

  - forward: the parallel direction (IAF sampling, MAF logpdf), one network evaluation
  - inverse: the sequential direction (MAF sampling), D rows one after another
  - VJP of each: x̄ and all four parameter cotangents (ȳ and l̄ given)

and, for the parallel direction, the MLP coupling with identical GEMM shapes -- COUPLING_MLP at chain dimension 2D with
n1 = n2 = D and the same H -- timed in the same round, alternating with the forward.

FMA per column: dense shapes 3·D·H (W₁ H x D, W₂ 2D x H); the entries the default MADE degrees leave unmasked are
counted from the masks.  The FMA bound uses the H100 SXM data-sheet FP32 rate (33.5 T FMA/s)."""
import argparse
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import autoregressive_oracle as A  # noqa: E402
import bijectors_jl_b200 as B  # noqa: E402
from bench_scale_matrix import PEAK_TFMAS, card, replay_median_ms  # noqa: E402
from bijectors_jl_b200.interface import _desc_array, _leaf_descs, _trainable_slots  # noqa: E402


def vjp_call(t, x, yb, lb, D, N, slot_floats):
    """One b2b_chain_vjp_f32 call of t with x̄ and every trainable cotangent, buffers allocated up front."""
    lib = B.lib()
    descs, _ = _leaf_descs(t, D, torch.float32)
    arr = _desc_array(descs)
    L = len(descs)
    bars = [torch.empty(slot_floats, device="cuda") if i in _trainable_slots(d) else None for d in descs for i in range(4)]
    ptrs = (ctypes.c_void_p * (4 * L))(*[None if b is None else b.data_ptr() for b in bars])
    xbar = B.colmajor_empty(D, N)
    ws_b = lib.b2b_chain_vjp_workspace_bytes(arr, L, D, N)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")

    def run():
        keep = (arr, bars, ptrs, xbar, ws)  # noqa: F841
        B._lib.check(lib.b2b_chain_vjp_f32(arr, L, x.data_ptr(), yb.data_ptr(), lb.data_ptr(), xbar.data_ptr(),
                                           ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b,
                                           torch.cuda.current_stream().cuda_stream), "b2b_chain_vjp_f32")

    return run


def bench(D, H, N, lines):
    rng = np.random.default_rng(D + H)
    W1 = (rng.standard_normal((H, D)) * 0.5 / np.sqrt(D)).astype(np.float32)
    W2 = (rng.standard_normal((2 * D, H)) * 0.5 / np.sqrt(H)).astype(np.float32)
    c1, c2 = (rng.standard_normal(H) * 0.1).astype(np.float32), (rng.standard_normal(2 * D) * 0.1).astype(np.float32)
    lay = B.MaskedAutoregressive(W1, c1, W2, c2)
    M1, M2 = A.masks(lay.degrees, D)
    used = int(M1.sum() + M2.sum())  # unmasked FMAs per column
    dense = 3 * D * H
    cpl = B.Coupling(B.MLPConditioner(W1, c1, W2, c2), B.PartitionMask(2 * D, list(range(1, D + 1)),
                                                                      list(range(D + 1, 2 * D + 1))))
    x = B.colmajor_empty(D, N)
    x.copy_(torch.randn((N, D), device="cuda").t())
    y = B.colmajor_empty(D, N)
    lj = torch.empty(N, device="cuda")
    yb = B.colmajor_empty(D, N)
    yb.copy_(torch.randn((N, D), device="cuda").t())
    lb = torch.ones(N, device="cuda")
    x2 = B.colmajor_empty(2 * D, N)
    x2.copy_(torch.randn((N, 2 * D), device="cuda").t())
    y2 = B.colmajor_empty(2 * D, N)
    cases = [
        ("forward", lambda: B.run_chain(lay, x, y=y, logjac=lj)),
        ("coupling 2D", lambda: B.run_chain(cpl, x2, y=y2, logjac=lj)),
        ("inverse", lambda: B.run_chain(B.inverse(lay), x, y=y, logjac=lj)),
        ("VJP forward", vjp_call(lay, x, yb, lb, D, N, 2 * D * H)),
        ("VJP inverse", vjp_call(B.inverse(lay), x, yb, lb, D, N, 2 * D * H)),
    ]
    times = {name: [] for name, _ in cases}
    for _ in range(3):
        for name, fn in cases:
            times[name].append(replay_median_ms(fn, reps=10))
    med = {name: float(np.median(v)) for name, v in times.items()}
    logn = int(np.log2(N))
    for name, _ in cases:
        t = med[name]
        fma = dense * (2 if name.startswith("VJP") else 1)  # the VJP: the forward network and its transpose, plus G
        tb = fma * N / (PEAK_TFMAS * 1e12) * 1e3
        rounds = ["%.3f" % v for v in times[name]]
        line = (f"{name:12s} D={D:4d} H={H:4d} N=2^{logn}  {t:9.3f} ms  {fma * N / t / 1e9:7.2f} T dense FMA/s"
                f"  ({tb / t * 100:5.1f} % of the FP32 FMA bound)  rounds {rounds}")
        print(line, flush=True)
        lines.append(line)
    line = (f"summary D={D} H={H}: FMA per column dense {dense}, unmasked {used} ({used / dense * 100:.0f} %);  forward / "
            f"coupling 2D {med['forward'] / med['coupling 2D']:.3f};  inverse / forward {med['inverse'] / med['forward']:.2f};"
            f"  VJP inverse / VJP forward {med['VJP inverse'] / med['VJP forward']:.2f}")
    print(line, flush=True)
    lines.append(line)
    del x, y, yb, x2, y2
    torch.cuda.empty_cache()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "bench_autoregressive_h100.txt"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    lines = [card()]
    print(lines[0], flush=True)
    for D in (16, 64, 128):
        for H in (64, 256):
            bench(D, H, 1 << 20, lines)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
