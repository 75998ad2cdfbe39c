"""Times the triangular Scale layer (B2B_SCALE_TRIANGULAR) at D = 64, 128, 256 and N = 2^20 with the method of
tools/bench_scale_matrix.py (device time of graph-captured calls, median of 20 replays, three rounds; the card and its power
limit read in the same run), and writes the table to --out (default records/bench_scale_triangular_h100.txt):

  - forward  y = T x, T = LowerTriangular   (prep launch, then the triangular map)
  - inverse  y = T⁻¹ x                        (prep launch forming T⁻¹, then the triangular map)
  - logpdf of transformed(MvNormal(μ, Diagonal(σ²)), Scale(T))   (the inverse layer, then the fused diagonal terminal)
  - VJP of the forward layer with x̄ and T̄ (ȳ and l̄ given)
  - the prep launch alone: the forward and the inverse call at N = 1
  - the LU pair Scale(UnitLowerTriangular(L)) ∘ Scale(UpperTriangular(U)) against the dense Scale(L·U), both directions

Bounds from the shape with H100 SXM data-sheet figures (33.5 T FP32 FMA/s, 3.35 TB/s): D(D+1)/2·N FMAs and (8D + 4)·N
bytes for the forward and inverse; D(D+1)·N FMAs and (12D + 4)·N bytes for the VJP of the forward layer (the transposed
triangular map and G on the triangle); for the LU pair twice the single layer's, for the dense layer D²·N FMAs."""
import argparse
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bijectors_jl_b200 as B  # noqa: E402
from bench_scale_matrix import bound_ms, card, replay_median_ms  # noqa: E402


def tri(rng, D, upper):
    T = 0.3 * rng.standard_normal((D, D)) / np.sqrt(D)
    T = np.triu(T, 1) if upper else np.tril(T, -1)
    return (T + np.diag(rng.uniform(0.5, 2.0, D) * np.where(rng.uniform(size=D) < 0.25, -1, 1))).astype(np.float32)


def bench(D, N, lines):
    rng = np.random.default_rng(D)
    Tl = tri(rng, D, False)
    lay = B.Scale(B.LowerTriangular(Tl))
    inv = B.inverse(lay)
    base = B.MvNormal(D, mu=(rng.standard_normal(D) * 0.3).astype(np.float32), sigma=rng.uniform(0.7, 1.3, D).astype(np.float32))
    td = B.transformed(base, lay)
    L, U = tri(rng, D, False), tri(rng, D, True)
    pair = B.Composed(B.Scale(B.UpperTriangular(U)), B.Scale(B.UnitLowerTriangular(L)))
    dense = B.Scale((np.tril(L, -1) + np.eye(D)) @ np.triu(U))
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
    tbar = torch.empty(D * D, device="cuda")
    ptrs = (ctypes.c_void_p * 4)(tbar.data_ptr())
    ws_b = lib.b2b_chain_vjp_workspace_bytes(arr, 1, D, N)
    ws = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731

    def vjp():
        B._lib.check(lib.b2b_chain_vjp_f32(arr, 1, x.data_ptr(), yb.data_ptr(), lb.data_ptr(), xbar.data_ptr(),
                                           ctypes.cast(ptrs, ctypes.c_void_p), D, N, D, D, D, ws.data_ptr(), ws_b, stream()),
                     "b2b_chain_vjp_f32")

    tri_fma = D * (D + 1) // 2
    cases = [
        ("forward", lambda: B.run_chain(lay, x, y=y, logjac=lj), bound_ms(8 * D + 4, tri_fma, N)),
        ("inverse", lambda: B.run_chain(inv, x, y=y, logjac=lj), bound_ms(8 * D + 4, tri_fma, N)),
        ("logpdf (diagonal base)", lambda: B.logpdf(td, x), bound_ms(8 * D + 4, tri_fma, N)),
        ("VJP (x̄, T̄)", vjp, bound_ms(12 * D + 4, 2 * tri_fma, N)),
        ("prep: forward, N = 1", lambda: B.run_chain(lay, x1, y=y1, logjac=lj1), None),
        ("prep: inverse, N = 1", lambda: B.run_chain(inv, x1, y=y1, logjac=lj1), None),
        ("LU pair forward", lambda: B.run_chain(pair, x, y=y, logjac=lj), bound_ms(16 * D + 8, 2 * tri_fma, N)),
        ("dense L·U forward", lambda: B.run_chain(dense, x, y=y, logjac=lj), bound_ms(8 * D + 4, D * D, N)),
        ("LU pair inverse", lambda: B.run_chain(B.inverse(pair), x, y=y, logjac=lj), bound_ms(16 * D + 8, 2 * tri_fma, N)),
        ("dense L·U inverse", lambda: B.run_chain(B.inverse(dense), x, y=y, logjac=lj), bound_ms(8 * D + 4, D * D, N)),
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
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "bench_scale_triangular_h100.txt"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    lines = [card()]
    print(lines[0], flush=True)
    for D in (64, 128, 256):
        bench(D, 1 << 20, lines)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
