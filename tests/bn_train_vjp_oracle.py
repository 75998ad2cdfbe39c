"""Float64 reference for the reverse mode of the training-mode InvertibleBatchNorm (normalise.jl:51-67 with istraining()
== true), restated from ``oracle_np.batchnorm_forward(..., training=True)``: m = mean(x), v = sum((x − m)²)/n over the
columns, y = A (x − m) + b with A = e^logs/√(v + eps), logjac = fill(Σ_c (logs_c − log(v_c + eps)/2), n).  With the
column sums S1 = Σȳ, S2 = Σȳ(x − m), L̄ = Σl̄ and σ² = v + eps:

    x̄    = A ȳ − A S1/n − (x − m)(A S2 + L̄)/(n σ²)
    b̄    = S1
    l̄ogs = A S2 + L̄

The last term of x̄ holds both the usual BatchNorm backward (m and v depend on x) and −L̄(x − m)/(nσ²), the log-Jacobian's
dependence on the batch variance.  The moving-statistics update has no cotangent.  Checked against central differences
of the forward in tests/test_batchnorm_train_vjp.py."""
import numpy as np


def batchnorm_train_vjp(bn, x, ybar, ljbar, stats=None):
    """(x̄ (C, N), b̄ (C,), l̄ogs (C,)) in x's dtype.  ``ybar`` / ``ljbar`` may be None (zeros).  ``stats`` = (m, v, n): the
    statistics of a larger batch this x is a column shard of -- x̄ then needs the sums S1, S2, L̄ of that whole batch, so
    only b̄ and l̄ogs (this shard's share) are returned with ``x̄ = None``; see ``batchnorm_train_vjp_shard``."""
    dt = x.dtype
    n = x.shape[-1]
    if stats is None:
        m = x.mean(axis=-1, keepdims=True)
        v = ((x - m) ** 2).sum(axis=-1, keepdims=True) / dt.type(n)
    else:
        m, v, n = np.asarray(stats[0], dt)[:, None], np.asarray(stats[1], dt)[:, None], stats[2]
    s2 = v + dt.type(bn.eps)
    A = np.exp(bn.logs.astype(dt))[:, None] / np.sqrt(s2)
    yb = np.zeros_like(x) if ybar is None else ybar.astype(dt)
    L = dt.type(0) if ljbar is None else ljbar.astype(dt).sum()
    S1 = yb.sum(axis=-1, keepdims=True)
    S2 = (yb * (x - m)).sum(axis=-1, keepdims=True)
    bbar, logsbar = S1[:, 0], (A * S2)[:, 0] + L
    if stats is not None:
        return None, bbar, logsbar
    xbar = A * yb - A * S1 / dt.type(n) - (x - m) * (A * S2 + L) / (dt.type(n) * s2)
    return xbar.astype(dt), bbar.astype(dt), logsbar.astype(dt)


def batchnorm_train_vjp_shard(bn, x, ybar, ljbar, lo, hi):
    """Columns lo:hi of the full-batch x̄, and the b̄ / l̄ogs summed over those columns only (what one rank of a sharded
    batch returns), with the full batch's statistics."""
    xbar, _, _ = batchnorm_train_vjp(bn, x, ybar, ljbar)
    m = x.mean(axis=-1)
    v = ((x - m[:, None]) ** 2).sum(axis=-1) / x.dtype.type(x.shape[-1])
    _, bb, lb = batchnorm_train_vjp(bn, x[:, lo:hi], None if ybar is None else ybar[:, lo:hi],
                                    None if ljbar is None else ljbar[lo:hi], stats=(m, v, x.shape[-1]))
    return xbar[:, lo:hi], bb, lb
