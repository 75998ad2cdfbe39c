#!/usr/bin/env python
"""Tiny invocation of every kernel family that is not in sanitize_smoke.py, for compute-sanitizer:
   compute-sanitizer --tool memcheck python tools/sanitize_vjp.py
reverse mode (radial both directions + mixed, coupling fast / generic, BatchNorm, RQS both directions, planar runs),
the in-kernel sampler, Float64 chains, Logit / Truncated blocks, exact-L planar programs, padded spline tables."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bijectors_jl_b200 as B

f32 = np.float32
rng = np.random.default_rng(0)


def dev(a):
    return B.from_numpy(np.asarray(a, f32))


def radial(D):
    return B.RadialLayer(rng.standard_normal(1).astype(f32), rng.standard_normal(1).astype(f32), rng.standard_normal(D).astype(f32))


def planar(D):
    return B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32), f32([0.1]))


for D, N in ((64, 777), (32, 1000), (128, 333), (10, 129)):
    x, yb = dev(rng.standard_normal((D, N))), dev(rng.standard_normal((D, N)))
    lb = torch.randn(N, device="cuda")
    ls = [radial(D) for _ in range(5)]
    B.radial_chain_vjp(B.Composed(*ls), x, yb, lb)
    B.radial_chain_vjp(B.inverse(B.Composed(*ls)), x, yb, lb)
    B.radial_chain_vjp(B.Composed(ls[0], B.inverse(ls[1]), ls[2]), x, yb, None)
    bn = B.InvertibleBatchNorm(b=np.zeros(D, f32), logs=np.zeros(D, f32), m=np.zeros(D, f32), v=np.ones(D, f32))
    B.batchnorm_vjp(bn, x, yb, lb)
    B.batchnorm_vjp(B.inverse(bn), x, yb, lb)
    for K in (8, 5, 32):
        sp = B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                       rng.standard_normal((D, K - 1)).astype(f32), 3.0)
        B.rqs_vjp(sp, x, yb, lb)
        B.rqs_vjp(B.inverse(sp), x, yb, lb)
        if D in (32, 64):
            B.with_logabsdet_jacobian(sp, x)
            B.with_logabsdet_jacobian(B.inverse(sp), x)
    for n1, idx in ((D // 2, False), (D // 2 - 1, True)):
        i1 = list(range(1, n1 + 1))
        i2 = list(range(n1 + 1, D + 1)) if not idx else (rng.permutation(np.arange(n1 + 1, D + 1))[: D - n1 - 1]).tolist()
        cl = B.Coupling(B.AffineConditioner((rng.standard_normal((2 * n1, len(i2))) * 0.1).astype(f32), np.zeros(2 * n1, f32)),
                        B.PartitionMask(D, i1, i2))
        B.coupling_vjp(cl, x, yb, lb)
        B.coupling_vjp(B.inverse(cl), x, yb, lb)
    if D in (32, 64, 128):
        for L in (3, 5, 7, 11):
            pl = [planar(D) for _ in range(L)]
            B.with_logabsdet_jacobian(B.Composed(*pl), x)
            B.with_logabsdet_jacobian(B.inverse(B.Composed(*pl)), x)
            B.logpdf(B.transformed(B.MvNormal(D), B.Composed(*pl)), x)
        pl = [planar(D) for _ in range(4)]
        B.planar_chain_vjp(B.Composed(pl[0], B.inverse(pl[1]), pl[2], pl[3]), x, yb, lb)
    td = B.transformed(B.MvNormal(D), B.Composed(planar(D), radial(D)))
    B.rand(td, 500, seed=3)
    x64 = B.from_numpy(rng.standard_normal((D, 200)), dtype=np.float64)
    B.with_logabsdet_jacobian(B.RadialLayer(np.array([0.2]), np.array([0.3]), rng.standard_normal(D), dtype=torch.float64), x64)
    torch.cuda.synchronize()
    print(f"D={D} N={N} ok")
xnd = torch.from_numpy(np.asfortranarray(rng.standard_normal((3, 4, 6, 17)).astype(f32))).cuda()
B.with_logabsdet_jacobian(B.InvertibleBatchNorm(6), xnd)
torch.cuda.synchronize()
print("done")
