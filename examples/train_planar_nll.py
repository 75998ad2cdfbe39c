"""The reference's flow-training example (docs/src/flows.md:40-110) on the H100 path: a PlanarLayer flow on 2-D data,
trained by gradient descent on the negative log-likelihood −Σ logpdf(transformed(MvNormal(2, 1), flow), data).
The reference differentiates with ForwardDiff; here torch.autograd drives b2b_planar_chain_vjp_f32 (reverse mode).

    python examples/train_planar_nll.py            # needs an H100 (no CPU fallback)
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bijectors_jl_b200 as B


def main(n_layers=1, n_points=1000, iters=1000, stepsize=1e-3):
    torch.manual_seed(0)
    D = 2
    flow = B.autograd.PlanarFlow(D, n_layers)                # PlanarLayer(2): randn-initialised w, u, b
    data = B.colmajor_empty(D, n_points)
    data.copy_(torch.randn(D, n_points, device="cuda"))       # xs = randn(2, 1000)

    def nll():
        x, logjac = flow.inverse(data)                        # logpdf(td, y) = logpdf(base, x) + logjac
        base = -0.5 * (x * x).sum(dim=0) - 0.5 * D * math.log(2 * math.pi)
        return -(base + logjac).sum()

    print(f"Initial loss = {float(nll().detach()):.4f}")
    opt = torch.optim.SGD(flow.parameters(), lr=stepsize)
    for _ in range(iters):
        opt.zero_grad()
        loss = nll()
        loss.backward()
        opt.step()
    print(f"Final loss = {float(nll().detach()):.4f}")
    td = B.transformed(B.MvNormal(D), B.Composed(*flow.layers()))
    samples = B.rand(td, 1000)
    print("sample mean", samples.mean(dim=1).tolist(), "sample var", samples.var(dim=1).tolist())


if __name__ == "__main__":
    main()
