"""Float64 reference of B2B_ELEMENTWISE_VEC: Shift(a), Scale(a) and LeakyReLU(a) with a vector a[D] (shift.jl, scale.jl:16,
31-32, leaky_relu.jl:25-29), one law on every row with the row's own parameter, either direction -- its map, per-column
log-Jacobian, and reverse mode to x and to a:

  law        forward y, ℓ                       ∂y/∂a, ∂ℓ/∂a        inverse y, ℓ              ∂y/∂a, ∂ℓ/∂a
  Shift      x + a, 0                           1, 0                x − a, 0                  −1, 0
  Scale      a·x, Σ log|a|                      x, 1/a              x/a, −Σ log|a|            −x/a², −1/a
  LeakyReLU  x < 0 ? a·x : x, Σ_{x<0} log a     x, 1/a (x < 0)      x < 0 ? x/a : x, −Σ log a  −x/a², −1/a (x < 0)

VecLayer evaluates in the dtype of its input (float32 gives the reference's own float32 error for the parity gates), and
plugs into tests/chain_vjp_oracle.py as a layer of kind "elementwise_vec"."""
from __future__ import annotations

import numpy as np

import chain_vjp_oracle as V
import mvnormal_tril_oracle as T

SHIFT, SCALE, LEAKY_RELU = 3, 4, 5  # B2B_EW_* of include/b2b.h


class VecLayer:
    kind = "elementwise_vec"

    def __init__(self, law: int, a):
        if law not in (SHIFT, SCALE, LEAKY_RELU):
            raise ValueError(law)
        self.law, self.a = law, np.asarray(a, np.float64)

    @property
    def name(self) -> str:
        """The reference's field name of the parameter: LeakyReLU's α, Shift's and Scale's a."""
        return "α" if self.law == LEAKY_RELU else "a"

    def _apply(self, x, inverse):
        x = np.asarray(x)
        a = self.a.astype(x.dtype)[:, None]
        if self.law == SHIFT:
            return (x - a if inverse else x + a), np.zeros(x.shape[1], x.dtype)
        mask = np.ones_like(x, bool) if self.law == SCALE else x < 0
        y = np.where(mask, x / a if inverse else a * x, x)
        lj = (np.log(np.abs(a)) * mask).sum(axis=0)
        return y, (-lj if inverse else lj).astype(x.dtype)

    def forward(self, x):
        return self._apply(x, False)

    def inverse(self, x):
        return self._apply(x, True)

    def vjp(self, x, ybar, ljbar, inverse=False):
        """(x̄, {name: ā}) of with_logabsdet_jacobian(layer or its inverse, x) with cotangents ȳ (D, N) and l̄ (N,)."""
        x = np.asarray(x)
        dt = x.dtype
        a = self.a.astype(dt)[:, None]
        ybar = np.zeros_like(x) if ybar is None else np.asarray(ybar, dt)
        lb = np.asarray(ljbar, dt)[None, :]
        if self.law == SHIFT:
            return ybar.copy(), {self.name: (ybar * (-1.0 if inverse else 1.0)).sum(axis=1)}
        mask = np.ones_like(x, bool) if self.law == SCALE else x < 0
        f = np.where(mask, 1 / a if inverse else a, 1.0)
        dy = np.where(mask, -x / (a * a) if inverse else x, 0.0)
        dl = np.where(mask, -1 / a if inverse else 1 / a, 0.0)
        return (ybar * f).astype(dt), {self.name: (ybar * dy + lb * dl).sum(axis=1).astype(dt)}


def chain_vjp(layers, inverse_flags, x, ybar, ljbar, mu=None, sigma=None, terminal=False, dtype=np.float64,
              scale_tril=None):
    """chain_vjp_oracle.chain_vjp (same arguments and results) for chains that also hold VecLayers: each VecLayer is
    differentiated by its own vjp, every other layer by the per-kind rules of tests/chain_vjp_oracle.py."""
    x = np.asarray(x, dtype)
    N = x.shape[1]
    lb = np.zeros(N, dtype) if ljbar is None else np.asarray(ljbar, dtype)
    inputs, cur = [], x
    for lay, inv in zip(layers, inverse_flags):
        inputs.append(cur)
        cur = (lay.inverse if inv else lay.forward)(cur)[0]
    g = np.zeros_like(cur) if ybar is None else np.asarray(ybar, dtype)
    base = {}
    if scale_tril is not None:
        gx, gm, gL = T.logpdf_vjp(scale_tril, mu, cur, lb, dtype)
        g = g + gx
        if mu is not None:
            base["μ"] = gm
        base["L"] = gL
    elif terminal:
        mu_, sigma_ = (None if v is None else np.asarray(v, dtype) for v in (mu, sigma))
        gx, gm, gs = V.mvnormal_diag_logpdf_vjp(mu_, sigma_, cur, lb)
        g = g + gx
        if mu is not None:
            base["μ"] = gm
        if sigma is not None:
            base["σ"] = gs
    grads = [None] * len(layers)
    for l in reversed(range(len(layers))):
        lay, inv = layers[l], inverse_flags[l]
        if isinstance(lay, VecLayer):
            g, grads[l] = lay.vjp(inputs[l], g, lb, inv)
        else:
            g, grads[l] = V._layer_vjp(lay, inv, inputs[l], g, lb)
    return g, grads, base
