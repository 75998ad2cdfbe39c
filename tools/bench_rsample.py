#!/usr/bin/env python
"""Reparameterised sampling against what it replaces, in one process with the two sides alternating:
  forward : rand(td, n, with_logjac=True)  vs  rand_logpdf(td, n)         (b2b_chain_sample_f32 vs _logq_f32)
  backward: b2b_randn_f32 + b2b_chain_vjp_f32 on a materialised x  vs  b2b_chain_sample_vjp_f32
on three chains: the C2 chain (8 x Planar, D = 128, N = 2^20), a RealNVP chain of COUPLING_MLP layers (D = 64) and an
8-layer planar chain over a full-covariance (TRIL) base at D = 128.  Bytes per sample are computed from the shapes.
    python tools/bench_rsample.py [--N 1048576] [--reps 20]"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B  # noqa: E402


def print_card():
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    print(f"card: {torch.cuda.get_device_name()}, power limit, max SM clock: {power}")


def time_pair(fa, fb, reps):
    """Median ms of fa and fb, measured alternately with CUDA events (each warmed up first)."""
    for f in (fa, fb, fa, fb):
        f()
    ta, tb = [], []
    for _ in range(reps):
        for f, t in ((fa, ta), (fb, tb)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            e.synchronize()
            t.append(s.elapsed_time(e))
    return float(np.median(ta)), float(np.median(tb))


def planar_chain(D, rng):
    return B.Composed(*[B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                      (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32),
                                      rng.standard_normal(1).astype(np.float32)) for _ in range(8)])


def realnvp(D, rng, blocks=4, H=64):
    n1 = D // 2
    layers = []
    for k in range(blocks):
        lo, hi = (range(1, n1 + 1), range(n1 + 1, D + 1)) if k % 2 == 0 else (range(n1 + 1, D + 1), range(1, n1 + 1))
        cond = B.MLPConditioner((rng.standard_normal((H, D - n1)) * 0.1).astype(np.float32), np.zeros(H, np.float32),
                                (rng.standard_normal((2 * n1, H)) * 0.01).astype(np.float32), np.zeros(2 * n1, np.float32))
        layers.append(B.Coupling(cond, B.PartitionMask(D, lo, hi)))
    return B.Composed(*layers)


def case(name, td, D, N, reps):
    seed = 1234
    ybar = B.colmajor_empty(D, N)
    ybar.normal_()
    lqbar = torch.randn(N, device="cuda")
    fa = lambda: B.rand(td, N, seed=seed, with_logjac=True)
    fb = lambda: B.rand_logpdf(td, N, seed=seed)
    ta, tb = time_pair(fa, fb, reps)
    ya, _ = fa()
    yb, _ = fb()
    same = bool(torch.equal(ya, yb))
    del ya, yb
    x = B.colmajor_empty(D, N)
    base = td.dist
    mu = base.mu.data_ptr() if base.mu is not None else None
    lib, stream = B.lib(), torch.cuda.current_stream().cuda_stream

    def materialised():
        # the base samples drawn straight into x (b2b_randn_f32, or the TRIL sample launch), then the chain's reverse mode
        if base._tril is not None:
            rc = lib.b2b_chain_sample_tril_f32(None, 0, mu, base._tril.data_ptr(), ctypes.c_uint64(seed), ctypes.c_uint64(0),
                                               0, x.data_ptr(), None, D, N, D, None, 0, stream)
        else:
            rc = lib.b2b_randn_f32(x.data_ptr(), mu, base.sigma.data_ptr() if base.sigma is not None else None,
                                   ctypes.c_uint64(seed), ctypes.c_uint64(0), 0, D, N, D, stream)
        assert rc == 0, rc
        B.chain_vjp(td.transform, x, ybar, -lqbar)

    fd = lambda: B.rand_vjp(td, N, ybar, lqbar, seed=seed)
    tc, td_ = time_pair(materialised, fd, reps)
    # bytes per sample moved by the forward's output (y and log q / logjac): identical for both entry points
    fwd_bytes = 4 * (D + 1)
    print(f"{name:34s} D={D:4d} N={N}  forward: rand(with_logjac) {ta:8.3f} ms   rand_logpdf {tb:8.3f} ms "
          f"({100 * (tb / ta - 1):+.1f} %)  {fwd_bytes} B/sample each, y bit-identical: {same}")
    print(f"{'':34s} backward: randn + chain_vjp {tc:8.3f} ms   rand_vjp (b2b_chain_sample_vjp_f32) {td_:8.3f} ms "
          f"({100 * (td_ / tc - 1):+.1f} %)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rsample.py measures on the GPU"
    print_card()
    rng = np.random.default_rng(0)
    D = 128
    case("C2: 8 x Planar, MvNormal(D)", B.transformed(B.MvNormal(D), planar_chain(D, rng)), D, a.N, a.reps)
    D = 64
    base = B.MvNormal(D, mu=np.zeros(D, np.float32), sigma=np.ones(D, np.float32))
    case("RealNVP, 4 x COUPLING_MLP (H=64)", B.transformed(base, realnvp(D, rng)), D, a.N, a.reps)
    D = 128
    Lf = (np.eye(D) + np.tril(rng.standard_normal((D, D)) * 0.02, -1)).astype(np.float32)
    base = B.MvNormal(D, mu=np.zeros(D, np.float32), scale_tril=Lf)
    case("8 x Planar over a TRIL base", B.transformed(base, planar_chain(D, rng)), D, a.N, a.reps)


if __name__ == "__main__":
    main()
