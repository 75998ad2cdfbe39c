"""Times the LU linear layer (B2B_SCALE_LU, LULinear(F, p)) at D = 64, 128, 256 and N = 2^20 with the method of
tools/bench_scale_matrix.py (device time of graph-captured calls, median of 20 replays, three rounds; the card and its power
limit read in the same run), and writes the table to --out (default records/bench_scale_lu_h100.txt).  In every round the
same call is timed for three layers on the same factors, one after another:

  - LULinear(F, p)                                                      (prep launch, then the dense map)
  - Permute(p) ∘ Scale(UnitLowerTriangular(F)) ∘ Scale(UpperTriangular(F))   (the three-layer composition)
  - Scale(A), A = P·L·U                                                 (the dense layer: LU of A, then the same map)

and the calls are: forward, inverse, logpdf of transformed(MvNormal(μ, Diagonal(σ²)), layer), and the VJP of the forward
layer with x̄ and every parameter cotangent (ȳ and l̄ given).

Bounds of LULinear from the shape with H100 SXM data-sheet figures (33.5 T FP32 FMA/s, 3.35 TB/s): D²·N FMAs and (8D + 4)·N
bytes for the forward, the inverse and the logpdf; 2·D²·N FMAs and (12D + 4)·N bytes for the VJP (the transposed map and
G).  The map column "map" is the forward's time less the prep launch alone (the forward at N = 1)."""
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
from bijectors_jl_b200.interface import _desc_array, _leaf_descs, _trainable_slots  # noqa: E402


def factors(rng, D):
    F = 0.3 * rng.standard_normal((D, D)) / np.sqrt(D)
    np.fill_diagonal(F, rng.uniform(0.5, 2.0, D) * np.where(rng.uniform(size=D) < 0.25, -1, 1))
    return F.astype(np.float32)


def vjp_call(t, x, yb, lb, D, N):
    """One b2b_chain_vjp_f32 call of the chain t with x̄ and every trainable cotangent, buffers allocated up front."""
    lib = B.lib()
    descs, _ = _leaf_descs(t, D, torch.float32)
    arr = _desc_array(descs)
    L = len(descs)
    bars = [torch.empty(D * D, device="cuda") if i in _trainable_slots(d) else None for d in descs for i in range(4)]
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


def bench(D, N, lines):
    rng = np.random.default_rng(D)
    F = factors(rng, D)
    p = rng.permutation(D) + 1
    lay = B.LULinear(F, p)
    comp = B.Composed(B.Scale(B.UpperTriangular(F)), B.Scale(B.UnitLowerTriangular(F)), B.Permute(p))
    A = np.zeros((D, D))
    A[p - 1] = (np.tril(F, -1) + np.eye(D)) @ np.triu(F)  # row r of L·U is row p[r] of A
    dense = B.Scale(A.astype(np.float32))
    mu = (rng.standard_normal(D) * 0.3).astype(np.float32)
    sigma = rng.uniform(0.7, 1.3, D).astype(np.float32)
    x = B.colmajor_empty(D, N)
    x.copy_(torch.randn((N, D), device="cuda").t())
    y = B.colmajor_empty(D, N)
    lj = torch.empty(N, device="cuda")
    yb = B.colmajor_empty(D, N)
    yb.copy_(torch.randn((N, D), device="cuda").t())
    lb = torch.ones(N, device="cuda")
    x1, y1, lj1 = B.colmajor_empty(D, 1), B.colmajor_empty(D, 1), torch.empty(1, device="cuda")
    x1.zero_()
    lu_fma, tri_fma = D * D, D * (D + 1) // 2
    layers = [("LULinear", lay), ("composition", comp), ("dense Scale(A)", dense)]
    cases = []
    for name, t in layers:
        td = B.transformed(B.MvNormal(D, mu=mu, sigma=sigma), t)
        bnd = name == "LULinear"
        cases += [
            (f"forward {name}", lambda t=t: B.run_chain(t, x, y=y, logjac=lj), bound_ms(8 * D + 4, lu_fma, N) if bnd else None),
            (f"inverse {name}", lambda t=t: B.run_chain(B.inverse(t), x, y=y, logjac=lj),
             bound_ms(8 * D + 4, lu_fma, N) if bnd else None),
            (f"logpdf {name}", lambda td=td: B.logpdf(td, x), bound_ms(8 * D + 4, lu_fma, N) if bnd else None),
            (f"VJP {name}", vjp_call(t, x, yb, lb, D, N), bound_ms(12 * D + 4, 2 * lu_fma, N) if bnd else None),
        ]
    cases += [("prep LULinear forward, N = 1", lambda: B.run_chain(lay, x1, y=y1, logjac=lj1), None),
              ("prep LULinear inverse, N = 1", lambda: B.run_chain(B.inverse(lay), x1, y=y1, logjac=lj1), None)]
    times = {name: [] for name, _, _ in cases}
    for _ in range(3):
        for name, fn, _ in cases:
            times[name].append(replay_median_ms(fn))
    med = {name: float(np.median(v)) for name, v in times.items()}
    logn = int(np.log2(N))
    for name, _, bnd in cases:
        t = med[name]
        rounds = ["%.3f" % v for v in times[name]]
        if name.startswith("prep"):
            line = f"{name:32s} D={D:4d}          {t:8.3f} ms  rounds {rounds}"
        elif bnd is None:
            line = f"{name:32s} D={D:4d} N=2^{logn}  {t:8.3f} ms  rounds {rounds}"
        else:
            tb, side = bnd
            line = (f"{name:32s} D={D:4d} N=2^{logn}  {t:8.3f} ms  bound {tb:6.3f} ms ({side})  {tb / t * 100:5.1f} % of bound"
                    f"  rounds {rounds}")
        print(line, flush=True)
        lines.append(line)
    fwd, inv, prep_f, prep_i = (med["forward LULinear"], med["inverse LULinear"], med["prep LULinear forward, N = 1"],
                                med["prep LULinear inverse, N = 1"])
    dense_map = med["forward dense Scale(A)"]
    line = (f"summary D={D}: LULinear / composition  forward {fwd / med['forward composition']:.2f}  inverse "
            f"{inv / med['inverse composition']:.2f}  logpdf {med['logpdf LULinear'] / med['logpdf composition']:.2f}  VJP "
            f"{med['VJP LULinear'] / med['VJP composition']:.2f};  LULinear / dense forward: forward {fwd / dense_map:.3f}"
            f"  inverse {inv / dense_map:.3f}  (map alone: {(fwd - prep_f) / dense_map:.3f}, {(inv - prep_i) / dense_map:.3f})")
    print(line, flush=True)
    lines.append(line)
    del x, y, yb
    torch.cuda.empty_cache()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "bench_scale_lu_h100.txt"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    lines = [card()]
    print(lines[0], flush=True)
    for D in (64, 128, 256):
        bench(D, 1 << 20, lines)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
