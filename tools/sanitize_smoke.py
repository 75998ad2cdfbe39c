#!/usr/bin/env python
"""Tiny invocation of every kernel family, meant to run under compute-sanitizer:
   compute-sanitizer --tool memcheck python tools/sanitize_smoke.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bijectors_jl_b200 as B

f32 = np.float32
rng = np.random.default_rng(0)


def run(D, N, variant):
    B.lib().b2b_set_kernel_variant(variant)
    n1 = D // 2
    layers = [
        B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32), f32([0.1])),
        B.InvertibleBatchNorm(b=np.zeros(D, f32), logs=np.zeros(D, f32), m=np.zeros(D, f32), v=np.ones(D, f32)),
        B.RadialLayer(f32([0.2]), f32([0.3]), rng.standard_normal(D).astype(f32)),
        B.RationalQuadraticSpline(rng.standard_normal((D, 8)).astype(f32), rng.standard_normal((D, 8)).astype(f32),
                                  rng.standard_normal((D, 7)).astype(f32), 3.0),
        B.Coupling(B.AffineConditioner((rng.standard_normal((2 * n1, D - n1)) * 0.1).astype(f32)),
                   B.PartitionMask(D, list(range(1, n1 + 1)), list(range(n1 + 1, D + 1)))),
        B.LeakyReLU(0.2),
        B.Permute((rng.permutation(D) + 1).tolist()),
    ]
    flow = B.Composed(*layers)
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    y, lj = B.with_logabsdet_jacobian(flow, x)
    xi, lji = B.with_logabsdet_jacobian(B.inverse(flow), y)
    td = B.transformed(B.MvNormal(D), flow)
    tot, lp = B.logpdf_sum(td, y)
    torch.cuda.synchronize()
    err = float((xi - x).norm() / x.norm())
    print(f"D={D} N={N} variant={variant}: roundtrip {err:.2e} total {float(tot):.4f}")
    assert err < 1e-3


for D, N in [(128, 200), (64, 100), (32, 70), (256, 130), (10, 50)]:
    for variant in (0, 1, 10):
        run(D, N, variant)
# constant-bank planar chains (device and host parameters, both directions, logpdf) and their reverse mode
B.lib().b2b_set_kernel_variant(0)
for D, L, N in [(128, 8, 333), (64, 3, 100), (32, 1, 70)]:
    pl = [B.PlanarLayer((rng.standard_normal(D) / np.sqrt(D)).astype(f32), (rng.standard_normal(D) / np.sqrt(D)).astype(f32),
                        rng.standard_normal(1).astype(f32)) for _ in range(L)]
    flow = B.Composed(*pl)
    x = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    y, lj = B.with_logabsdet_jacobian(flow, x)
    xi, _ = B.with_logabsdet_jacobian(B.inverse(flow), y)
    yh, _ = B.with_logabsdet_jacobian(B.Composed(*[l.to("cpu") for l in pl]), x)
    B.logpdf_sum(B.transformed(B.MvNormal(D), flow), y)
    yb = B.from_numpy(rng.standard_normal((D, N)).astype(f32))
    lb = torch.randn(N, device="cuda")
    B.planar_chain_vjp(flow, x, yb, lb)
    B.planar_chain_vjp(B.inverse(flow), y, yb, lb)
    torch.cuda.synchronize()
    assert float((xi - x).norm() / x.norm()) < 1e-3 and float((yh - y).norm() / y.norm()) < 1e-5
    print(f"planar const / vjp D={D} L={L} ok")
rf = B.Composed(*[B.RadialLayer(f32([0.2]), f32([0.3]), rng.standard_normal(64).astype(f32)) for _ in range(3)])
B.radial_chain_vjp(rf, B.from_numpy(rng.standard_normal((64, 211)).astype(f32)), B.from_numpy(rng.standard_normal((64, 211)).astype(f32)), torch.randn(211, device="cuda"))
torch.cuda.synchronize()
print("radial vjp ok")
bn = B.InvertibleBatchNorm(32, training=True)
bn.train_forward(B.from_numpy(rng.standard_normal((32, 300)).astype(f32)))
xh = B.from_numpy(rng.standard_normal((64, 1000)).astype(f32), device="cpu", pin_memory=True)
B.with_logabsdet_jacobian(B.PlanarLayer(64), xh)
torch.cuda.synchronize()
print("sanitize smoke done")
