"""TransformedDistribution on the device path (src/transformed_distribution.jl).

  TransformedDistribution(dist, transform) / transformed(d, b)   :9-17, :37-38
  logpdf(td, y::Matrix) = logpdf(td.dist, x) + logjac with
      (x, logjac) = with_logabsdet_jacobian(inverse(td.transform), y)          :165-169
  rand(td, n): base samples pushed through the forward chain                   :212-224
  rand_logpdf / rand_vjp: the reparameterised sampler of variational inference   :210-213 (docs/src/advi.md)

The inverse chain, the base MvNormal log-density and (optionally) the batch sum run as ONE fused chain
launch per fusable segment: the terminal B2B_MVNORMAL_DIAG op consumes the recovered x in registers, so no
D×N intermediate is ever written.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import _lib
from .interface import Transform, _batch_view, inverse, run_chain
from .layers import _desc, _dev_f32


class PosDefException(ValueError):
    """A covariance matrix whose Cholesky factorisation fails (LinearAlgebra's PosDefException, raised by PDMats)."""


class MvNormal:
    """MvNormal(μ, Diagonal(σ²)) / MvNormal(zeros(D), I) / MvNormal(μ, Σ) (Distributions + PDMats; third-party arithmetic
    restated in the kernels).

    * ``sigma``: the std-dev vector of a diagonal covariance, −(D·log2π + Σ log σ²)/2 − Σ((x−μ)/σ)²/2 (B2B_MVNORMAL_DIAG).
    * ``cov``: a dense D × D covariance Σ -- Distributions' FullNormal.  It is factorised once, in float64, into its lower
      Cholesky factor L (what the PDMat holds); a matrix that is not positive definite raises PosDefException.
    * ``scale_tril``: that factor L directly (lower triangle read, diagonal > 0), which is what a trainable base needs.
      −D·log2π/2 − Σ log Lᵢᵢ − ‖L⁻¹(x−μ)‖²/2 (B2B_MVNORMAL_TRIL): Float32 up to D = 256, Float64 up to D = 2048 (no
      Float64 sampler: ``rand`` raises TypeError).

    At most one of ``sigma``, ``cov`` and ``scale_tril`` may be given."""

    def __init__(self, D: int, mu=None, sigma=None, *, cov=None, scale_tril=None, device="cuda", dtype=torch.float32):
        if sum(v is not None for v in (sigma, cov, scale_tril)) > 1:
            raise ValueError("MvNormal: give at most one of sigma, cov and scale_tril")
        self.D = int(D)
        self.dtype = dtype
        self.mu = None if mu is None else _dev_f32(mu, device, dtype)
        self.sigma = None if sigma is None else _dev_f32(sigma, device, dtype)
        self.device = device
        for t in (self.mu, self.sigma):
            if t is not None and t.numel() != self.D:
                raise ValueError("DimensionMismatch: MvNormal parameter length")
        if cov is not None:
            c = torch.as_tensor(np.asarray(cov.detach().cpu() if isinstance(cov, torch.Tensor) else cov, np.float64))
            if c.shape != (self.D, self.D):
                raise ValueError(f"DimensionMismatch: covariance of shape {tuple(c.shape)} for a {self.D}-dim MvNormal")
            scale_tril, info = torch.linalg.cholesky_ex(c)
            if int(info) != 0:
                raise PosDefException(f"matrix is not positive definite; Cholesky factorization failed (leading minor "
                                      f"{int(info)})")
        # L is held column-major -- the layout the library reads -- as the row-major D × D tensor Lᵀ
        self._tril = None
        if scale_tril is not None:
            L = scale_tril.detach() if isinstance(scale_tril, torch.Tensor) else torch.as_tensor(np.asarray(scale_tril))
            if tuple(L.shape) != (self.D, self.D):
                raise ValueError(f"DimensionMismatch: scale_tril of shape {tuple(L.shape)} for a {self.D}-dim MvNormal")
            self._tril = L.to(device=device, dtype=dtype).t().contiguous()

    @property
    def scale_tril(self) -> Optional[torch.Tensor]:
        """The lower Cholesky factor L (a view of the device storage), or None for a diagonal covariance."""
        return None if self._tril is None else self._tril.t()

    def __len__(self):
        return self.D

    def _terminal_desc(self):
        if self._tril is not None:
            return _desc(_lib.MVNORMAL_TRIL, False, p0=self.mu, p1=self._tril)
        return _desc(_lib.MVNORMAL_DIAG, False, p0=self.mu if self.mu is not None else None,
                     p1=self.sigma if self.sigma is not None else None, _f64=self.dtype == torch.float64)

    def rand(self, n: int, seed: Optional[int] = None, offset: int = 0, column_offset: int = 0) -> torch.Tensor:
        """D×n base samples mu + sigma .* z, or mu + L z (column-major), from the library's Philox4x32-10 + Box-Muller
        stream (b2b_randn_f32): a pure function of (seed, offset, global column, row)."""
        return _sample(self, (), n, seed, offset, column_offset, want_logjac=False)[0]


class _Identity(Transform):
    def _descs(self, inverse_, D, dtype=torch.float32):
        return []


class TransformedDistribution:
    """struct TransformedDistribution{D,B} (transformed_distribution.jl:9-17)."""

    def __init__(self, dist: MvNormal, transform: Transform):
        self.dist, self.transform = dist, transform

    def __len__(self):
        return len(self.dist)


def transformed(d: MvNormal, b: Transform) -> TransformedDistribution:
    """transformed(d, b) (transformed_distribution.jl:37-38)."""
    return TransformedDistribution(d, b)


def logpdf(td, y: torch.Tensor) -> torch.Tensor:
    """logpdf(td::MvTransformed, y::Matrix) -> N-vector (transformed_distribution.jl:165-169);
    logpdf(d::MvNormal, x) for a bare base distribution."""
    if isinstance(td, MvNormal):
        return run_chain(_Identity(), y, want_y=False, extra_descs=[td._terminal_desc()])[1]
    D, _, _ = _batch_view(y)
    if D != len(td.dist):
        raise ValueError(f"DimensionMismatch: distribution has {len(td.dist)} dims, input has {D}")
    inv = inverse(td.transform)
    return run_chain(inv, y, want_y=False, extra_descs=[td.dist._terminal_desc()])[1]


def logpdf_sum(td, y: torch.Tensor, out: Optional[torch.Tensor] = None):
    """(Σ_n logpdf(td, y_n) as a device float64 scalar, logpdf vector): the training objective of
    docs/src/flows.md:74-77, reduced on the device in a fixed order."""
    if out is None:
        out = torch.zeros((), dtype=torch.float64, device=y.device if y.is_cuda else "cpu")
    if isinstance(td, MvNormal):
        t, term = _Identity(), td._terminal_desc()
    else:
        t, term = inverse(td.transform), td.dist._terminal_desc()
    _, lp = run_chain(t, y, want_y=False, extra_descs=[term], sum_out=out)
    return out, lp


def _seed(seed: Optional[int]) -> int:
    """Explicit seed, or one drawn from torch's default CPU generator (so torch.manual_seed makes sampling reproducible,
    the role `rng` plays in rand(rng, td, n))."""
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    return int(seed) & 0xFFFFFFFFFFFFFFFF


def _sample(dist: MvNormal, transform, n: int, seed, offset, column_offset, want_logjac):
    from ._lib import check, lib
    from .interface import _desc_array, _stream, colmajor_empty

    import ctypes

    if dist._tril is not None and dist.dtype != torch.float32:
        raise TypeError("rand: a Float64 full-covariance MvNormal has no device sampler (construct it with dtype=torch.float32)")
    D = dist.D
    if isinstance(transform, tuple):
        descs = list(transform)
    else:
        descs = list(transform._descs(False, D, torch.float32))
    L = len(descs)
    arr = _desc_array(descs) if L else None
    dev = dist.device if not isinstance(dist.device, str) or dist.device != "cuda" else torch.device("cuda", torch.cuda.current_device())
    y = colmajor_empty(D, n, dev)
    lj = torch.empty((n,), dtype=torch.float32, device=y.device) if want_logjac else None
    ws_bytes = lib().b2b_chain_workspace_bytes(arr, L, D, n, 1, 0) if L else 0
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=y.device) if ws_bytes else None
    if dist._tril is not None:
        rc = lib().b2b_chain_sample_tril_f32(
            arr, L, dist.mu.data_ptr() if dist.mu is not None else None, dist._tril.data_ptr(),
            ctypes.c_uint64(_seed(seed)), ctypes.c_uint64(int(offset)), int(column_offset), y.data_ptr(),
            lj.data_ptr() if lj is not None else None, D, n, D, ws.data_ptr() if ws is not None else None, ws_bytes,
            _stream())
        check(rc, "b2b_chain_sample_tril_f32")
        return y, lj
    rc = lib().b2b_chain_sample_f32(
        arr, L, dist.mu.data_ptr() if dist.mu is not None else None, dist.sigma.data_ptr() if dist.sigma is not None else None,
        ctypes.c_uint64(_seed(seed)), ctypes.c_uint64(int(offset)), int(column_offset), y.data_ptr(),
        lj.data_ptr() if lj is not None else None, D, n, D, ws.data_ptr() if ws is not None else None, ws_bytes, _stream())
    check(rc, "b2b_chain_sample_f32")
    return y, lj


def rand(td, n: int, seed: Optional[int] = None, offset: int = 0, column_offset: int = 0, with_logjac: bool = False):
    """rand(rng, td, n) (transformed_distribution.jl:212-224): base samples pushed through the forward chain.  The
    reference draws z on the host and maps the transform over the columns one by one; here the normals are generated
    INSIDE the chain kernel (b2b_chain_sample_f32: Philox4x32-10 + Box-Muller), so the D×n base samples never exist in
    device memory.  `seed` plays the role of `rng` (default: drawn from torch's generator); `column_offset` lets a
    column shard continue ONE global stream (rank r passes the index of its first column).  `with_logjac=True` also
    returns log|det J| of the transform at the samples."""
    if isinstance(td, MvNormal):
        y, lj = _sample(td, (), n, seed, offset, column_offset, with_logjac)
    else:
        y, lj = _sample(td.dist, td.transform, n, seed, offset, column_offset, with_logjac)
    return (y, lj) if with_logjac else y


def logpdf_vjp(td: TransformedDistribution, y: torch.Tensor, lpbar: Optional[torch.Tensor] = None):
    """Reverse mode of ``logpdf(td, y)``: one b2b_chain_vjp_f32 call (b2b_chain_vjp_f64 for a Float64 ``y``, with Float64
    layers and base) through inverse(td.transform) and the terminal MvNormal.  ``lpbar`` (N, None = ones in ``y``'s dtype)
    is the cotangent of the logpdf vector.  Returns ``(ybar, flow_grads, base_grads)``:
    ``flow_grads`` one dict per leaf of ``flatten(td.transform)`` in FLOW order (see chain_vjp for the keys) and
    ``base_grads`` = {"μ", "σ"} (or {"μ", "L"} for a full-covariance base, L̄ lower triangular) for the base parameters
    that are given; all summed over the columns of this batch."""
    from .interface import _chain_vjp_raw, _leaf_descs, _leaf_grads, _slot_grads, _trainable_slots

    D, N, _ = _batch_view(y)
    if D != len(td.dist):
        raise ValueError(f"DimensionMismatch: distribution has {len(td.dist)} dims, input has {D}")
    if lpbar is None:
        lpbar = torch.ones((N,), dtype=y.dtype, device=y.device)
    descs, counts = _leaf_descs(inverse(td.transform), D, y.dtype)
    descs.append(td.dist._terminal_desc())
    want = [(l, i) for l, d in enumerate(descs) for i in _trainable_slots(d)]
    ybar, bars = _chain_vjp_raw(descs, y, None, lpbar, want)
    flow = _leaf_grads(descs, counts, bars)[::-1]
    T = len(descs) - 1
    return ybar, flow, _slot_grads(descs[T], T, bars)


def _rsample_setup(td, n: int, where: str):
    """(base MvNormal, descriptors of the forward chain, per-leaf descriptor counts, base descriptor, device) of the
    reparameterised sampler, after the argument checks that need no device: Float32 only (TypeError otherwise)."""
    from .interface import _leaf_descs

    dist, t = (td, None) if isinstance(td, MvNormal) else (td.dist, td.transform)
    if not isinstance(dist, MvNormal):
        raise TypeError(f"{where}: the base must be an MvNormal, got {type(dist).__name__}")
    if dist.dtype != torch.float32:
        raise TypeError(f"{where}: the sampler is Float32 only (construct the base with dtype=torch.float32)")
    if int(n) < 0:
        raise ValueError(f"{where}: n must be >= 0")
    descs, counts = _leaf_descs(t, dist.D, torch.float32) if t is not None else ([], [])
    dev = dist.device if not isinstance(dist.device, str) or dist.device != "cuda" else torch.device("cuda", torch.cuda.current_device())
    return dist, descs, counts, dist._terminal_desc(), dev


def rand_logpdf(td, n: int, seed: Optional[int] = None, offset: int = 0, column_offset: int = 0):
    """``(y, logq)``: the samples ``rand(td, n, seed, offset, column_offset)`` draws -- bit for bit -- and their
    log-density log q(y) = logpdf(td, y), formed in the same pass from the base draw z and the forward log-Jacobian
    (b2b_chain_sample_logq_f32): log q = −½‖z‖² − Σ log σᵢ (or log Lᵢᵢ) − ½·D·log2π − ℓ(x).  No inverse chain runs,
    so it costs what ``rand(with_logjac=True)`` costs.  Float32 flows and bases only (TypeError otherwise)."""
    import ctypes

    from ._lib import check, lib
    from .interface import _desc_array, _stream, colmajor_empty

    dist, descs, _, base, dev = _rsample_setup(td, n, "rand_logpdf")
    D, L = dist.D, len(descs)
    arr = _desc_array(descs) if L else None
    bdesc = _desc_array([base])
    y = colmajor_empty(D, n, dev)
    lq = torch.empty((n,), dtype=torch.float32, device=y.device)
    ws_bytes = lib().b2b_chain_sample_logq_workspace_bytes(arr, L, bdesc, D, n)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=y.device) if ws_bytes else None
    rc = lib().b2b_chain_sample_logq_f32(arr, L, bdesc, ctypes.c_uint64(_seed(seed)), ctypes.c_uint64(int(offset)),
                                         int(column_offset), y.data_ptr(), lq.data_ptr(), D, n, D,
                                         ws.data_ptr() if ws is not None else None, ws_bytes, _stream())
    check(rc, "b2b_chain_sample_logq_f32")
    return y, lq


def _rand_vjp_raw(descs, base, D: int, n: int, dev, ybar, lqbar, seed: int, offset: int, column_offset: int, want):
    """One b2b_chain_sample_vjp_f32 call.  ``descs`` + [``base``] index the cotangents; ``want``: (descriptor index, slot)
    pairs.  Returns {(l, i): cotangent in the storage shape of that parameter}."""
    import ctypes

    from ._lib import check, lib
    from .interface import _batch_view, _desc_array, _slot_shape, _stream

    L = len(descs)
    ldyb = D
    if ybar is not None:
        Dy, Ny, ldyb = _batch_view(ybar)
        if (Dy, Ny) != (D, n) or not ybar.is_cuda or ybar.dtype != torch.float32:
            raise ValueError("rand_vjp: ybar must be a Float32 device batch of the samples' shape")
    if lqbar is not None and (lqbar.numel() != n or lqbar.dtype != torch.float32 or not lqbar.is_contiguous()):
        raise ValueError("rand_vjp: lqbar must be a contiguous float32 vector of length n")
    arr = _desc_array(descs) if L else None
    bdesc = _desc_array([base])
    full = list(descs) + [base]
    bars = {}
    ptrs = (ctypes.c_void_p * (4 * (L + 1)))()
    for l, i in want:
        t = torch.empty(_slot_shape(full[l], i, D), dtype=torch.float32, device=dev)
        bars[(l, i)] = t
        ptrs[4 * l + i] = t.data_ptr()
    L_ = lib()
    ws_bytes = L_.b2b_chain_sample_vjp_workspace_bytes(arr, L, bdesc, D, n)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
    rc = L_.b2b_chain_sample_vjp_f32(arr, L, bdesc, ctypes.c_uint64(seed), ctypes.c_uint64(int(offset)),
                                     int(column_offset), ybar.data_ptr() if ybar is not None else None, ldyb,
                                     lqbar.data_ptr() if lqbar is not None else None, ptrs, D, n,
                                     ws.data_ptr() if ws is not None else None, ws_bytes, _stream())
    check(rc, "b2b_chain_sample_vjp_f32")
    return bars


def rand_vjp(td, n: int, ybar: Optional[torch.Tensor] = None, lqbar: Optional[torch.Tensor] = None,
             seed: Optional[int] = None, offset: int = 0, column_offset: int = 0):
    """Reverse mode of ``rand_logpdf(td, n, seed, offset, column_offset)`` with the base draw z held fixed -- the
    reparameterisation gradient of an ELBO: one b2b_chain_sample_vjp_f32 call.  ``ybar`` (D×n) and ``lqbar`` (n) are the
    cotangents of the samples and of log q (None = zeros); pass the ``seed`` the forward used.  Returns ``(flow_grads,
    base_grads)`` with the shapes and leaf order of ``logpdf_vjp``: one dict per leaf of ``flatten(td.transform)`` and
    {"μ", "σ"} (or {"μ", "L"}, L̄ lower triangular) for the base parameters that are given, summed over the n columns."""
    from .interface import _leaf_grads, _slot_grads, _trainable_slots

    if seed is None:
        raise ValueError("rand_vjp: pass the seed the samples were drawn with")
    dist, descs, counts, base, dev = _rsample_setup(td, n, "rand_vjp")
    full = list(descs) + [base]
    want = [(l, i) for l, d in enumerate(full) for i in _trainable_slots(d)]
    bars = _rand_vjp_raw(descs, base, dist.D, int(n), dev, ybar, lqbar, _seed(seed), offset, column_offset, want)
    T = len(descs)
    return _leaf_grads(descs, counts, bars), _slot_grads(base, T, bars)
