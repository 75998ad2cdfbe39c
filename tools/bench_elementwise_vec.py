#!/usr/bin/env python
"""Vector Shift / Scale (B2B_ELEMENTWISE_VEC) against the STACKED_EW layers they equal, in one process with the sides
alternating (CUDA-event medians):
  VJP    : b2b_chain_vjp_f32 of [Scale(a), Shift(b), MvNormal diag] at D = 128, N = 2^22 with l̄ given (ȳ = 0): the
           STACKED_EW chain, the vector chain x̄ only, and the vector chain with ā and b̄ (the SLOTS instantiation)
  forward: with_logabsdet_jacobian of Shift(b) ∘ Scale(a) ∘ 4 x Planar, one fused launch, against its STACKED_EW form
Bytes are computed from the shapes: the VJP reads x and l̄ and writes x̄ (8·D + 4 bytes a column), the forward reads x and
writes y and logjac (8·D + 4).  The HBM-bound fraction is the bytes over the time, divided by the rate of a device-to-device
copy of the same number of bytes measured in the same process.
    python tools/bench_elementwise_vec.py [--D 128] [--N 4194304] [--reps 20]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B  # noqa: E402
from bijectors_jl_b200.interface import _chain_vjp_raw, _leaf_descs  # noqa: E402
from bijectors_jl_b200.layers import _desc  # noqa: E402


def print_card():
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    print(f"card: {torch.cuda.get_device_name()}, power limit, max SM clock: {power}")


def time_all(fs, reps):
    """Median ms of each callable, measured round-robin with CUDA events after a warm-up of each."""
    for f in fs + fs:
        f()
    ts = [[] for _ in fs]
    for _ in range(reps):
        for f, t in zip(fs, ts):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            e.synchronize()
            t.append(s.elapsed_time(e))
    return [float(np.median(t)) for t in ts]


class StackedEq(B.Transform):
    """The STACKED_EW layer equal to a vector Shift / Scale: code[r] = its law, the same parameter tensor."""

    def __init__(self, lay):
        self.lay = lay
        self.code = torch.full((lay.a.numel(),), lay.code, dtype=torch.int32, device=lay.a.device)

    def _descs(self, inverse, D, dtype=torch.float32):
        return [_desc(B._lib.STACKED_EW, inverse, i0=self.code, p0=self.lay.a)]

    def _keepalive(self):
        return (self.code, self.lay.a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--D", type=int, default=128)
    ap.add_argument("--N", type=int, default=1 << 22)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    D, N = a.D, a.N
    print(f"# tools/bench_elementwise_vec.py (D = {D}, N = {N}, {a.reps} round-robin repetitions, CUDA-event medians)")
    print_card()
    rng = np.random.default_rng(0)
    s = B.Scale(rng.uniform(0.5, 2.0, D).astype(np.float32))
    t = B.Shift(rng.standard_normal(D).astype(np.float32))
    x = B.colmajor_empty(D, N)
    x.normal_()
    lb = torch.randn(N, device="cuda")
    nbytes = (8 * D + 4) * N
    src = torch.empty(nbytes // 4, device="cuda")
    dst = torch.empty_like(src)
    copy_ms = time_all([lambda: dst.copy_(src)], a.reps)[0]
    copy_rate = 2 * nbytes / copy_ms / 1e6  # a copy reads and writes: GB/s
    print(f"device-to-device copy of {nbytes / 2**20:.0f} MiB: {copy_ms:.3f} ms, {copy_rate:.0f} GB/s (read + write)")

    term = B.MvNormal(D)._terminal_desc()
    chains = {"STACKED_EW": B.Composed(StackedEq(s), StackedEq(t)), "vector": B.Composed(s, t)}
    descs = {k: _leaf_descs(c, D)[0] + [term] for k, c in chains.items()}
    runs = {
        "STACKED_EW, x̄": lambda: _chain_vjp_raw(descs["STACKED_EW"], x, None, lb, []),
        "vector, x̄ only": lambda: _chain_vjp_raw(descs["vector"], x, None, lb, []),
        "vector, x̄ + ā + b̄": lambda: _chain_vjp_raw(descs["vector"], x, None, lb, [(0, 0), (1, 0)]),
    }
    xb = {k: f()[0] for k, f in runs.items()}
    same = all(torch.equal(xb["STACKED_EW, x̄"], v) for v in xb.values())
    ms = time_all(list(runs.values()), a.reps)
    print(f"VJP [Scale(a), Shift(b), MvNormal diag]  {8 * D + 4} B/column, x̄ bit-identical across the three: {same}")
    for (k, _), m in zip(runs.items(), ms):
        rate = nbytes / m / 1e6
        print(f"  {k:<22} {m:8.3f} ms  {rate:6.0f} GB/s  {rate / copy_rate * 100:5.1f} % of the copy rate")
    del xb

    pls = [B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                         (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32), rng.standard_normal(1).astype(np.float32))
           for _ in range(4)]
    fwd = {"STACKED_EW": B.Composed(*pls, StackedEq(s), StackedEq(t)), "vector": B.Composed(*pls, s, t)}
    y = {k: B.colmajor_empty(D, N) for k in fwd}
    fs = [lambda k=k: B.with_logabsdet_jacobian_(fwd[k], x, y[k], None) for k in fwd]
    outs = [f() for f in fs]
    same = torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    ms = time_all(fs, a.reps)
    print(f"forward Shift(b) ∘ Scale(a) ∘ 4 x Planar, one fused launch, {8 * D + 4} B/column, y and logjac bit-identical: {same}")
    for k, m in zip(fwd, ms):
        rate = nbytes / m / 1e6
        print(f"  {k:<22} {m:8.3f} ms  {rate:6.0f} GB/s  {rate / copy_rate * 100:5.1f} % of the copy rate")


if __name__ == "__main__":
    main()
