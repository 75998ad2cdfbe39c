"""Host-side mirror of Bijectors.jl's Transform interface (src/interface.jl) for the batched device path.

Same names, argument meaning and error behaviour as the reference:
  Transform / Bijector / Inverse            src/interface.jl:133,246-271
  transform, logabsdetjac,
  with_logabsdet_jacobian (+ in-place "!")  src/interface.jl:144,156-166,183-192,212-218
  inverse                                   src/interface.jl:265-266
  ∘ (here `@` or compose(...)), Composed    Base.ComposedFunction + src/bijectors/composed.jl
  default inverse log-Jacobian              src/interface.jl:276-281 (fused on the device)

Batches are Julia-layout column-major ``D×N`` Float32 matrices: a torch tensor of shape ``(D, N)`` with
strides ``(1, D)`` (see :func:`colmajor_empty` / :func:`from_numpy`).  A 1-D tensor of length D is a single
column.  Device tensors take the device entry points; host (CPU) tensors take the chunked
host-buffer entry point ``b2b_chain_run_host_f32`` and return host tensors.  All arithmetic happens in
libb2b.so -- this module only builds layer descriptors and launches.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import B2BError, LayerDesc, check, lib

# --------------------------------------------------------------------------------------------------
# layout helpers
# --------------------------------------------------------------------------------------------------


def colmajor_empty(D: int, N: int, device="cuda", dtype=torch.float32, pin_memory=False) -> torch.Tensor:
    """Uninitialised Julia-layout (column-major) D×N matrix: shape (D, N), strides (1, D)."""
    if pin_memory:
        base = torch.empty((N, D), dtype=dtype, pin_memory=True)
    else:
        base = torch.empty((N, D), dtype=dtype, device=device)
    return base.t()


def from_numpy(a: np.ndarray, device="cuda", pin_memory=False, dtype=np.float32) -> torch.Tensor:
    """numpy (D, N) or (D,) array -> Julia-layout tensor on ``device`` (Float32 by default, dtype=np.float64 for the
    Float64 path)."""
    a = np.asarray(a, dtype=dtype)
    if a.ndim == 1:
        t = torch.from_numpy(np.ascontiguousarray(a))
        return t.pin_memory() if (pin_memory and device == "cpu") else t.to(device)
    base = torch.from_numpy(np.ascontiguousarray(a.T))  # (N, D) row-major == (D, N) column-major
    if device == "cpu":
        return (base.pin_memory() if pin_memory else base).t()
    return base.to(device).t()


def to_numpy(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().numpy()


def _batch_view(x: torch.Tensor) -> Tuple[int, int, int]:
    """(D, N, ld) of a column batch; raises like a Julia MethodError for anything else."""
    if x.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"batches are Float32 (hot path) or Float64 (b2b_chain_run_f64), got {x.dtype}")
    if x.dim() == 1:
        if x.stride(0) != 1:
            raise ValueError("vector input must be contiguous")
        return x.shape[0], 1, x.shape[0]
    if x.dim() != 2:
        raise ValueError(f"expected a D×N matrix or a length-D vector, got {tuple(x.shape)}")
    D, N = x.shape
    if N == 1:
        return D, 1, D
    if (D > 1 and x.stride(0) != 1) or x.stride(1) < D:  # the stride of a size-1 dimension is arbitrary
        raise ValueError(
            "batch must be Julia-layout column-major (shape (D, N), strides (1, ld>=D)); "
            "use colmajor_empty / from_numpy, or `x.t().contiguous().t()`"
        )
    return D, N, x.stride(1)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


# --------------------------------------------------------------------------------------------------
# Transform hierarchy
# --------------------------------------------------------------------------------------------------


class Transform:
    """abstract type Transform (src/interface.jl:133); callable: (t::Transform)(x) = transform(t, x) (:135)."""

    def __call__(self, x):
        return transform(self, x)

    # `outer @ inner` plays the role of `outer ∘ inner`
    def __matmul__(self, inner):
        return ComposedFunction(self, inner)

    def _descs(self, inverse: bool, D: int) -> List[LayerDesc]:
        raise NotImplementedError(
            f"`transform` not implemented for {type(self).__name__}; implement `transform` and/or "
            "`with_logabsdet_jacobian`."  # src/interface.jl:159-163
        )

    def _keepalive(self):
        return ()


class Bijector(Transform):
    """abstract type Bijector <: Transform (src/interface.jl:271)."""


class Inverse(Transform):
    """Inverse(orig) (src/interface.jl:246-266); with_logabsdet_jacobian(Inverse(b), y) =
    (x, -logabsdetjac(b, x)) (:278-281) is evaluated by ONE fused kernel per layer."""

    def __init__(self, orig: Transform):
        if not isinstance(orig, Transform):
            raise TypeError(f"{orig} is not invertible")
        self.orig = orig

    def _descs(self, inverse, D, dtype=torch.float32):
        return self.orig._descs(not inverse, D, dtype)

    def _keepalive(self):
        return self.orig._keepalive()

    def __eq__(self, other):
        return isinstance(other, Inverse) and self.orig == other.orig


def inverse(t):
    """inverse(t::Transform) = Inverse(t); inverse(ib::Inverse) = ib.orig (src/interface.jl:265-266);
    inverse(f∘g) = inverse(g) ∘ inverse(f) (InverseFunctions)."""
    if isinstance(t, Inverse):
        return t.orig
    if isinstance(t, ComposedFunction):
        return ComposedFunction(inverse(t.inner), inverse(t.outer))
    if isinstance(t, Composed):
        return Composed(*[inverse(b) for b in reversed(t.layers)])
    if hasattr(t, "_inverse"):
        return t._inverse()
    return Inverse(t)


class ComposedFunction(Transform):
    """outer ∘ inner (Base.ComposedFunction; methods in src/bijectors/composed.jl)."""

    def __init__(self, outer, inner):
        self.outer, self.inner = outer, inner

    def _descs(self, inverse_, D, dtype=torch.float32):
        # inverse(f∘g) = inverse(g)∘inverse(f): the outer function's inverse is applied first.  Every leaf inverts by
        # the descriptor's `inverse` flag on ITS OWN (cached) device tables -- no temporary objects whose device memory
        # could be recycled before the launch is enqueued.
        if inverse_:
            return self.outer._descs(True, D, dtype) + self.inner._descs(True, D, dtype)
        return self.inner._descs(False, D, dtype) + self.outer._descs(False, D, dtype)

    def _keepalive(self):
        return tuple(self.inner._keepalive()) + tuple(self.outer._keepalive())


class Composed(Transform):
    """Flat chain: Composed(L1, L2, ..., Ln) applies L1 first (== Ln ∘ … ∘ L1).  Accepts `∘` trees and
    flattens them (SURVEY Appendix C.1)."""

    def __init__(self, *layers):
        flat = []
        for b in layers:
            flat.extend(flatten(b))
        self.layers = flat

    def _descs(self, inverse_, D, dtype=torch.float32):
        out = []
        for b in (reversed(self.layers) if inverse_ else self.layers):
            out.extend(b._descs(inverse_, D, dtype))
        return out

    def _keepalive(self):
        return tuple(k for b in self.layers for k in b._keepalive())

    def to(self, device):
        """Functors.fmap-style movement of every layer that owns device tensors."""
        return Composed(*[b.to(device) if hasattr(b, "to") else b for b in self.layers])


class Columnwise(Transform):
    """columnwise(f) = Base.Fix1(eachcolmaphcat, f) (src/interface.jl:41,71-78): `f` applied to every column; its
    `logabsdetjac` / `with_logabsdet_jacobian` return the SUM of the per-column log-Jacobians (interface.jl:75-78).
    On the device the batched kernels already work column by column, so this only adds the fixed-order batch sum
    (returned as a float64 device scalar)."""

    def __init__(self, f):
        self.x = f  # Fix1 field name

    def _descs(self, inverse_, D, dtype=torch.float32):
        return self.x._descs(inverse_, D, dtype)

    def _keepalive(self):
        return self.x._keepalive()

    def _inverse(self):
        return Columnwise(inverse(self.x))  # inverse(f::Columnwise) = columnwise(inverse(f.x)), interface.jl:72


def columnwise(f):
    return Columnwise(f)


def compose(*fs):
    """compose(fn, ..., f2, f1) == fn ∘ … ∘ f2 ∘ f1."""
    out = fs[-1]
    for f in reversed(fs[:-1]):
        out = ComposedFunction(f, out)
    return out


def flatten(t) -> list:
    """Leaves of a `∘` tree in application order (inner-most first)."""
    if isinstance(t, ComposedFunction):
        return flatten(t.inner) + flatten(t.outer)
    if isinstance(t, Composed):
        return list(t.layers)
    return [t]


# --------------------------------------------------------------------------------------------------
# chain execution
# --------------------------------------------------------------------------------------------------

_HOST_CTX = {}


def _host_ctx(D: int, chunk_cols: int, n_streams: int):
    key = (torch.cuda.current_device(), chunk_cols, n_streams)
    ent = _HOST_CTX.get(key)
    if ent is None or ent[1] < D:
        if ent is not None:
            lib().b2b_host_ctx_destroy(ent[0])
        h = ctypes.c_void_p()
        check(lib().b2b_host_ctx_create(ctypes.byref(h), max(D, 1), chunk_cols, n_streams), "b2b_host_ctx_create")
        ent = (h, D)
        _HOST_CTX[key] = ent
    return ent[0]


HOST_CHUNK_COLS = 1 << 16
HOST_STREAMS = 3


def _desc_array(descs: Sequence[LayerDesc]):
    if len(descs) > _lib.MAX_CHAIN:
        raise B2BError(_lib.B2B_EUNSUPPORTED, f"chain of {len(descs)} layers (max {_lib.MAX_CHAIN})")
    return (LayerDesc * len(descs))(*descs)


def run_chain(t, x: torch.Tensor, *, want_y=True, want_logjac=True, y: Optional[torch.Tensor] = None,
              logjac: Optional[torch.Tensor] = None, accumulate=False, sum_out: Optional[torch.Tensor] = None,
              extra_descs: Sequence[LayerDesc] = (), keepalive=()):
    """Evaluate transform ``t`` (any Transform / chain) on batch ``x``.  Returns (y, logjac)."""
    D, N, ldx = _batch_view(x)
    descs = list(t._descs(False, D, x.dtype)) + list(extra_descs)
    if not descs:
        raise ValueError("empty chain")
    if x.dtype == torch.float64:
        return _run_chain_f64(descs, x, D, N, ldx, want_y, want_logjac, y, logjac, accumulate, sum_out)
    if any(hasattr(d, "_host_planar") for d in descs):
        return _run_planar_hostparams(descs, x, D, N, ldx, want_y, want_logjac, y, logjac, accumulate, sum_out)
    arr = _desc_array(descs)
    L = len(descs)
    if x.is_cuda:  # raw parameter pointers are launched on x's device: they must live there
        for kt in t._keepalive():
            if isinstance(kt, torch.Tensor) and kt.is_cuda and kt.device != x.device:
                raise ValueError(f"layer parameters live on {kt.device} but the batch is on {x.device}; move the flow with .to()")
    if not x.is_cuda:
        return _run_chain_host(arr, L, x, D, N, want_y, want_logjac, sum_out)
    L_ = lib()
    if want_y:
        if y is None:
            y = torch.empty_like(x) if x.dim() == 1 else colmajor_empty(D, N, x.device)
        Dy, Ny, ldy = _batch_view(y)
        if (Dy, Ny) != (D, N) or not y.is_cuda:
            raise ValueError("output shape mismatch")
    else:
        y, ldy = None, D
    if want_logjac or sum_out is not None:
        if logjac is None:
            logjac = torch.empty((N,), dtype=torch.float32, device=x.device)
        elif logjac.numel() != N or logjac.dtype != torch.float32 or not logjac.is_contiguous():
            raise ValueError("logjac must be a contiguous float32 vector of length N")
    else:
        logjac = None
    ws_bytes = L_.b2b_chain_workspace_bytes(arr, L, D, N, 1 if want_y else 0, 1 if sum_out is not None else 0)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device) if ws_bytes else None
    rc = L_.b2b_chain_run_f32(
        arr, L, x.data_ptr(), y.data_ptr() if y is not None else None,
        logjac.data_ptr() if logjac is not None else None,
        sum_out.data_ptr() if sum_out is not None else None,
        D, N, ldx, ldy, 1 if accumulate else 0,
        ws.data_ptr() if ws is not None else None, ws_bytes, _stream())
    check(rc, "b2b_chain_run_f32")
    lj_out = logjac
    if lj_out is not None and x.dim() == 1:
        lj_out = lj_out.reshape(())
    return y, lj_out


def _run_chain_f64(descs, x, D, N, ldx, want_y, want_logjac, y, logjac, accumulate, sum_out):
    """Float64 batches: b2b_chain_run_f64 (every layer kind; a correctness path, not the hot path).  Host tensors make
    the round trip through device memory here -- the computation itself always runs on the device."""
    if not all(isinstance(d, _lib.LayerDesc64) for d in descs):
        raise TypeError("Float64 batch with Float32 layer parameters: construct the layers with dtype=torch.float64")
    if len(descs) > _lib.MAX_CHAIN:
        raise B2BError(_lib.B2B_EUNSUPPORTED, f"chain of {len(descs)} layers (max {_lib.MAX_CHAIN})")
    if not x.is_cuda:
        if not torch.cuda.is_available():
            raise B2BError(_lib.B2B_EUNSUPPORTED, "no CUDA device: bijectors.jl_b200 has no CPU fallback")
        if sum_out is not None:
            raise B2BError(_lib.B2B_EUNSUPPORTED, "batch sums of Float64 host tensors: move the batch to the device")
        xd = x.cuda()
        yd, ld_ = _run_chain_f64(descs, xd, D, N, _batch_view(xd)[2], want_y, want_logjac, None, None, False, None)
        return (yd.cpu() if yd is not None else None), (ld_.cpu() if ld_ is not None else None)
    arr = (_lib.LayerDesc64 * len(descs))(*descs)
    L = len(descs)
    if want_y:
        if y is None:
            y = torch.empty_like(x) if x.dim() == 1 else colmajor_empty(D, N, x.device, dtype=torch.float64)
        ldy = _batch_view(y)[2]
    else:
        y, ldy = None, D
    if want_logjac or sum_out is not None:
        if logjac is None:
            logjac = torch.empty((N,), dtype=torch.float64, device=x.device)
    else:
        logjac = None
    L_ = lib()
    ws_bytes = L_.b2b_chain_workspace_bytes_f64(L, 1 if sum_out is not None else 0)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device) if ws_bytes else None
    rc = L_.b2b_chain_run_f64(arr, L, x.data_ptr(), y.data_ptr() if y is not None else None,
                              logjac.data_ptr() if logjac is not None else None,
                              sum_out.data_ptr() if sum_out is not None else None, D, N, ldx, ldy, 1 if accumulate else 0,
                              ws.data_ptr() if ws is not None else None, ws_bytes, _stream())
    check(rc, "b2b_chain_run_f64")
    if logjac is not None and x.dim() == 1:
        logjac = logjac.reshape(())
    return y, logjac


_HOSTPARAM_CACHE: dict = {}


def _run_planar_hostparams(descs, x, D, N, ldx, want_y, want_logjac, y, logjac, accumulate, sum_out):
    """∘-chains of PlanarLayers whose parameters are HOST tensors, on a device batch:
    b2b_planar_chain_hostparams_f32 (parameters travel as kernel arguments, include/b2b.h)."""
    if not all(hasattr(d, "_host_planar") for d in descs):
        raise B2BError(_lib.B2B_EUNSUPPORTED,
                       "mixed parameter residency: host-resident parameters are supported for chains made of "
                       "PlanarLayers only; move the flow to the device with .to('cuda')")
    inv = {int(d.inverse) for d in descs}
    if len(inv) != 1 or sum_out is not None or not x.is_cuda or x.dim() != 2:
        raise B2BError(_lib.B2B_EUNSUPPORTED,
                       "host-parameter planar chains take a device matrix, one direction, no batch sum; "
                       "move the flow to the device with .to('cuda')")
    L = len(descs)
    # L x D parameter blocks in application order; cached per (tensor identity, version) -- a few KB of host memory
    key = tuple((id(t), t._version) for d in descs for t in d._host_planar)
    packed = _HOSTPARAM_CACHE.get(key)
    if packed is None:
        if len(_HOSTPARAM_CACHE) >= 16:
            _HOSTPARAM_CACHE.clear()
        packed = (torch.stack([d._host_planar[0] for d in descs]).contiguous(),
                  torch.stack([d._host_planar[1] for d in descs]).contiguous(),
                  torch.stack([d._host_planar[2].reshape(-1)[0] for d in descs]).contiguous(),
                  [d._host_planar for d in descs])  # keeps the keyed tensors alive
        _HOSTPARAM_CACHE[key] = packed
    w, u, b = packed[0], packed[1], packed[2]
    if want_y:
        if y is None:
            y = colmajor_empty(D, N, x.device)
        Dy, Ny, ldy = _batch_view(y)
        if (Dy, Ny) != (D, N) or not y.is_cuda:
            raise ValueError("output shape mismatch")
    else:
        y, ldy = None, D
    if want_logjac:
        if logjac is None:
            logjac = torch.empty((N,), dtype=torch.float32, device=x.device)
        elif logjac.numel() != N or logjac.dtype != torch.float32 or not logjac.is_contiguous():
            raise ValueError("logjac must be a contiguous float32 vector of length N")
    else:
        logjac = None
    rc = lib().b2b_planar_chain_hostparams_f32(
        w.data_ptr(), u.data_ptr(), b.data_ptr(), L, inv.pop(), x.data_ptr(),
        y.data_ptr() if y is not None else None, logjac.data_ptr() if logjac is not None else None,
        D, N, ldx, ldy, 1 if accumulate else 0, _stream())
    check(rc, "b2b_planar_chain_hostparams_f32")
    return y, logjac


def _run_chain_host(arr, L, x, D, N, want_y, want_logjac, sum_out):
    """Host tensors: b2b_chain_run_host_f32 (chunked H2D/compute/D2H pipeline)."""
    if not torch.cuda.is_available():
        raise B2BError(_lib.B2B_EUNSUPPORTED, "no CUDA device: bijectors.jl_b200 has no CPU fallback")
    if x.dim() == 2 and N > 1 and x.stride(1) != D:
        raise ValueError("host batches must be dense column-major (ld == D)")
    ctx = _host_ctx(D, HOST_CHUNK_COLS, HOST_STREAMS)
    check(lib().b2b_host_ctx_wait_stream(ctx, _stream()), "b2b_host_ctx_wait_stream")  # parameters written on torch's stream
    pin = x.is_pinned()
    y = None
    if want_y:
        y = torch.empty_like(x) if x.dim() == 1 else colmajor_empty(D, N, "cpu", pin_memory=pin)
    lj = None
    if want_logjac:
        lj = torch.empty((N,), dtype=torch.float32, pin_memory=pin)
    hs = ctypes.c_double(0.0)
    rc = lib().b2b_chain_run_host_f32(
        ctx, arr, L, x.data_ptr(), y.data_ptr() if y is not None else None,
        lj.data_ptr() if lj is not None else None,
        ctypes.byref(hs) if sum_out is not None else None, D, N)
    check(rc, "b2b_chain_run_host_f32")
    if sum_out is not None:
        sum_out.fill_(hs.value)
    if lj is not None and x.dim() == 1:
        lj = lj.reshape(())
    return y, lj


class GraphedCalls:
    """A fixed sequence of chain launches captured ONCE into a CUDA graph and replayed with one graph launch.

    Every entry point of libb2b.so is launch-only on the caller's stream (no host synchronisation, no library-owned
    device state), so it is stream-capture safe; for launch-bound work -- a short spline pass on one shard of an 8-way
    sharded batch costs less GPU time than the Python + driver launch path -- replaying a captured graph removes the
    per-launch host cost (SURVEY §8(b): "graph-captured sequence").  `fn` must issue the same launches on the same
    buffers every time (shapes, pointers and parameters tensors are baked into the graph; parameter VALUES are read at
    replay time because they stay in device memory)."""

    def __init__(self, fn, warmup: int = 2):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):  # loads modules / sets function attributes outside the capture
                fn()
        torch.cuda.current_stream().wait_stream(s)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            fn()

    def __call__(self):
        self.graph.replay()


# --------------------------------------------------------------------------------------------------
# generic functions (src/interface.jl)
# --------------------------------------------------------------------------------------------------


def _batchnorm_nd(t, x, want_y=True, want_logjac=True):
    """InvertibleBatchNorm (or its Inverse) on an array of more than two dimensions (normalise.jl:41-47,61-67,74-86): the
    channel axis is ndims − 1, the batch axis the last one; ``x`` is Julia-layout (column-major, dense) with shape
    (d₁, …, d_k, C, B).  The slab of one batch element is a column of S·C numbers (S = d₁⋯d_k) whose row s + S·c belongs
    to channel c, so the elementwise map is the D×N kernel on a view of the same memory with each channel's parameters
    repeated S times; the log-Jacobian the reference returns -- fill(sum(logs − log(v + eps)/2), B), without a factor S
    (:66) -- is the C-channel layer's own log-Jacobian, evaluated by the library on a C×B batch."""
    inv = isinstance(t, Inverse)
    bn = t.orig if inv else t
    if getattr(bn, "training", False):
        raise B2BError(_lib.B2B_EUNSUPPORTED, "training-mode InvertibleBatchNorm takes D×N batches on the device path")
    shape = tuple(x.shape)
    C, Bn = shape[-2], shape[-1]
    if C != bn.b.numel():
        raise RuntimeError(f"InvertibleBatchNorm expected {bn.b.numel()} channels, got {C}")  # normalise.jl:43-45
    S = 1
    for d in shape[:-2]:
        S *= d
    strides, acc = [], 1
    for d in shape:
        strides.append(acc)
        acc *= d
    if tuple(x.stride()) != tuple(strides) or not x.is_cuda or x.dtype != bn.b.dtype:
        raise ValueError("arrays of more than two dimensions must be dense Julia-layout (column-major) device tensors "
                         "of the layer's element type")
    y = lj = None
    if want_y:
        wide = bn._expanded(S)
        y2 = run_chain(Inverse(wide) if inv else wide, x.as_strided((S * C, Bn), (1, S * C)), want_logjac=False)[0]
        y = y2.as_strided(shape, tuple(strides))
    if want_logjac:
        probe = torch.zeros((Bn, C), dtype=x.dtype, device=x.device).t()
        lj = run_chain(t, probe, want_y=False)[1]
    return y, lj


def _is_batchnorm_nd(t, x):
    from .layers import InvertibleBatchNorm
    base = t.orig if isinstance(t, Inverse) else t
    return isinstance(x, torch.Tensor) and x.dim() > 2 and isinstance(base, InvertibleBatchNorm)


def with_logabsdet_jacobian(t, x):
    """(transform(t, x), logabsdetjac(t, x)) in one fused pass (src/interface.jl:144)."""
    if _is_batchnorm_nd(t, x):
        return _batchnorm_nd(t, x)
    if hasattr(t, "_host_wladj") and not (isinstance(x, torch.Tensor) and x.is_cuda):
        return t._host_wladj(x)
    if isinstance(t, Columnwise):
        total = torch.zeros((), dtype=torch.float64, device=x.device if x.is_cuda else "cpu")
        y, _ = run_chain(t, x, sum_out=total)
        return y, total
    if getattr(t, "training", False) and hasattr(t, "train_forward"):  # istraining() == true, normalise.jl:51-60
        return t.train_forward(x)
    return run_chain(t, x)


def transform(t, x):
    """transform(b, x) (src/interface.jl:156-166)."""
    if _is_batchnorm_nd(t, x):
        return _batchnorm_nd(t, x, want_logjac=False)[0]
    if hasattr(t, "_host_wladj") and not (isinstance(x, torch.Tensor) and x.is_cuda):
        return t._host_wladj(x)[0]
    return run_chain(t, x, want_logjac=False)[0]


def logabsdetjac(t, x):
    """logabsdetjac(b, x) (src/interface.jl:183-192): no D×N store is issued."""
    if _is_batchnorm_nd(t, x):
        return _batchnorm_nd(t, x, want_y=False)[1]
    if hasattr(t, "_host_wladj") and not (isinstance(x, torch.Tensor) and x.is_cuda):
        return t._host_wladj(x)[1]
    if isinstance(t, Columnwise):  # sum over columns, interface.jl:75-77
        total = torch.zeros((), dtype=torch.float64, device=x.device if x.is_cuda else "cpu")
        run_chain(t, x, want_y=False, sum_out=total)
        return total
    return run_chain(t, x, want_y=False)[1]


def transform_(t, x, y=None):
    """transform!(b, x[, y]) (src/interface.jl:175-176): y defaults to x (in place)."""
    return run_chain(t, x, want_logjac=False, y=x if y is None else y)[0]


def with_logabsdet_jacobian_(t, x, y=None, logjac=None):
    """with_logabsdet_jacobian!(b, x[, y, logjac]) (src/interface.jl:212-218): returns
    (y, logjac + logjac_) with y defaulting to x."""
    return run_chain(t, x, y=x if y is None else y, logjac=logjac, accumulate=logjac is not None)


def logabsdetjac_(t, x, logjac=None):
    """logabsdetjac!(b, x[, logjac]) (src/interface.jl:199-200)."""
    return run_chain(t, x, want_y=False, logjac=logjac, accumulate=logjac is not None)[1]


class _DescSegment(Transform):
    """A run of already-built layer descriptors (a slice of a flattened chain)."""

    def __init__(self, descs, keep):
        self._d, self._k = list(descs), keep

    def _descs(self, inverse, D, dtype=torch.float32):
        if inverse:
            raise B2BError(_lib.B2B_EUNSUPPORTED, "internal segment: not invertible")
        return self._d

    def _keepalive(self):
        return self._k


def _direction_runs(descs, max_len: int = 8):
    """Cut a flattened chain into maximal runs of one direction (all forward / all Inverse) of at most `max_len` layers."""
    runs = []
    for d in descs:
        if runs and int(runs[-1][0].inverse) == int(d.inverse) and len(runs[-1]) < max_len:
            runs[-1].append(d)
        else:
            runs.append([d])
    return runs


def _planar_segment_vjp(descs, x, ybar, ljbar, want_param_grads):
    """One call of b2b_planar_chain_vjp_f32: <= 8 PlanarLayers, all forward or all Inverse."""
    D, N, ldx = _batch_view(x)
    ldyb = _batch_view(ybar)[2]
    L = len(descs)
    arr = _desc_array(descs)
    xbar = colmajor_empty(D, N, x.device)
    wbar = ubar = bbar = None
    if want_param_grads:
        wbar = torch.empty((L, D), dtype=torch.float32, device=x.device)
        ubar = torch.empty((L, D), dtype=torch.float32, device=x.device)
        bbar = torch.empty((L,), dtype=torch.float32, device=x.device)
    L_ = lib()
    ws_bytes = L_.b2b_planar_chain_vjp_workspace_bytes(L, D, N)
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=x.device)
    rc = L_.b2b_planar_chain_vjp_f32(
        arr, L, x.data_ptr(), ybar.data_ptr(), ljbar.data_ptr() if ljbar is not None else None, xbar.data_ptr(),
        wbar.data_ptr() if wbar is not None else None, ubar.data_ptr() if ubar is not None else None,
        bbar.data_ptr() if bbar is not None else None, D, N, ldx, ldyb, _batch_view(xbar)[2],
        ws.data_ptr(), ws_bytes, _stream())
    check(rc, "b2b_planar_chain_vjp_f32")
    grads = None
    if want_param_grads:
        grads = [{"w": wbar[l], "u": ubar[l], "b": bbar[l:l + 1]} for l in range(L)]
    return xbar, grads


def planar_chain_vjp(t, x: torch.Tensor, ybar: torch.Tensor, ljbar: Optional[torch.Tensor] = None,
                     want_param_grads: bool = True):
    """Vector-Jacobian product of ``with_logabsdet_jacobian(t, x)`` for a ∘-chain ``t`` of PlanarLayers:
    what the reference's reverse-mode AD computes in a training step (docs/src/flows.md:93-100,
    ext/BijectorsChainRulesCoreExt.jl).  ``ybar`` (D×N) / ``ljbar`` (N) are the cotangents of the two outputs.

    ``t`` may also be ``inverse(flow)`` (the chain ``logpdf(transformed(d, flow), y)`` evaluates,
    docs/src/flows.md:66-100): ``x`` is then the observed batch and ``find_alpha`` is differentiated with the reference's
    implicit-function rule (ext/BijectorsChainRulesCoreExt.jl:42-46).

    The device entry point differentiates up to 8 layers of ONE direction per call.  Longer chains and chains that mix
    PlanarLayers with Inverse(PlanarLayer)s are cut into such runs here: the run inputs are recomputed with the forward
    kernels, then the runs are differentiated last to first (the log-Jacobians add up, so every run sees the same l̄).

    Returns ``(xbar, grads)``: ``xbar`` (D×N) and ``grads`` = list of ``{"w": …, "u": …, "b": …}``, one entry per layer
    in APPLICATION order (``flatten(t)``; for ``inverse(flow)`` that is the flow's layers reversed), summed over the
    columns of this batch -- or ``None`` when ``want_param_grads`` is false."""
    D, N, ldx = _batch_view(x)
    Dy, Ny, ldyb = _batch_view(ybar)
    if (Dy, Ny) != (D, N) or not x.is_cuda or not ybar.is_cuda or x.dim() != 2:
        raise ValueError("planar_chain_vjp: x and ybar must be device matrices of the same D×N shape")
    descs = list(t._descs(False, D, x.dtype))
    if not descs or any(d.kind != _lib.PLANAR or hasattr(d, "_host_planar") for d in descs):
        raise B2BError(_lib.B2B_EUNSUPPORTED, "planar_chain_vjp: PlanarLayers (or their Inverses) with device parameters")
    if ljbar is not None and (ljbar.numel() != N or ljbar.dtype != torch.float32 or not ljbar.is_contiguous()):
        raise ValueError("ljbar must be a contiguous float32 vector of length N")
    runs = _direction_runs(descs)
    if len(runs) == 1:
        return _planar_segment_vjp(descs, x, ybar, ljbar, want_param_grads)
    keep = t._keepalive()
    inputs = [x]
    for r in runs[:-1]:
        inputs.append(run_chain(_DescSegment(r, keep), inputs[-1], want_logjac=False)[0])
    cot, grads = ybar, []
    for r, xin in zip(reversed(runs), reversed(inputs)):
        cot, g = _planar_segment_vjp(r, xin, cot, ljbar, want_param_grads)
        if want_param_grads:
            grads = g + grads
    return cot, (grads if want_param_grads else None)


def radial_chain_vjp(t, x: torch.Tensor, ybar: torch.Tensor, ljbar: Optional[torch.Tensor] = None):
    """Vector-Jacobian product of ``with_logabsdet_jacobian(t, x)`` for a ∘-chain ``t`` of (≤ 8) RadialLayers, D ≤ 128 --
    a flow, ``inverse(flow)`` (the logpdf / NLL path; ``x`` is then the observed batch) or a mix of directions.  Returns
    ``(xbar, grads)`` with ``grads`` = list of ``{"α_": …, "β": …, "z_0": …}`` per layer in APPLICATION order (cotangents of
    the RAW parameters, summed over the columns)."""
    D, N, ldx = _batch_view(x)
    Dy, Ny, ldyb = _batch_view(ybar)
    if (Dy, Ny) != (D, N) or not x.is_cuda or not ybar.is_cuda or x.dim() != 2:
        raise ValueError("radial_chain_vjp: x and ybar must be device matrices of the same D×N shape")
    descs = list(t._descs(False, D, x.dtype))
    if any(d.kind != _lib.RADIAL for d in descs):
        raise B2BError(_lib.B2B_EUNSUPPORTED, "radial_chain_vjp: RadialLayers (forward, Inverse, or mixed)")
    L = len(descs)
    arr = _desc_array(descs)
    if ljbar is not None and (ljbar.numel() != N or ljbar.dtype != torch.float32 or not ljbar.is_contiguous()):
        raise ValueError("ljbar must be a contiguous float32 vector of length N")
    xbar = colmajor_empty(D, N, x.device)
    abar = torch.empty((L,), dtype=torch.float32, device=x.device)
    bbar = torch.empty((L,), dtype=torch.float32, device=x.device)
    zbar = torch.empty((L, D), dtype=torch.float32, device=x.device)
    L_ = lib()
    ws_bytes = L_.b2b_radial_chain_vjp_workspace_bytes(L, D)
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=x.device)
    rc = L_.b2b_radial_chain_vjp_f32(
        arr, L, x.data_ptr(), ybar.data_ptr(), ljbar.data_ptr() if ljbar is not None else None, xbar.data_ptr(),
        abar.data_ptr(), bbar.data_ptr(), zbar.data_ptr(), D, N, ldx, ldyb, _batch_view(xbar)[2],
        ws.data_ptr(), ws_bytes, _stream())
    check(rc, "b2b_radial_chain_vjp_f32")
    return xbar, [{"α_": abar[l:l + 1], "β": bbar[l:l + 1], "z_0": zbar[l]} for l in range(L)]


def _layer_vjp(t, x, ybar, ljbar, kind, which):
    D, N, ldx = _batch_view(x)
    Dy, Ny, ldyb = _batch_view(ybar)
    if (Dy, Ny) != (D, N) or not x.is_cuda or not ybar.is_cuda or x.dim() != 2 or x.dtype != torch.float32:
        raise ValueError(f"{which}: x and ybar must be Float32 device matrices of the same D×N shape")
    descs = list(t._descs(False, D, torch.float32))
    if len(descs) != 1 or descs[0].kind != kind:
        raise B2BError(_lib.B2B_EUNSUPPORTED, f"{which}: one layer of the matching kind (or its Inverse)")
    if ljbar is not None and (ljbar.numel() != N or ljbar.dtype != torch.float32 or not ljbar.is_contiguous()):
        raise ValueError("ljbar must be a contiguous float32 vector of length N")
    return descs[0], D, N, ldx, ldyb


def coupling_vjp(t, x: torch.Tensor, ybar: torch.Tensor, ljbar: Optional[torch.Tensor] = None):
    """Vector-Jacobian product of ``with_logabsdet_jacobian(t, x)`` for ONE affine Coupling layer ``t`` (or
    ``inverse(coupling)``, with ``x`` the observed batch): b2b_coupling_affine_vjp_f32.  Returns ``(xbar, {"W": W̄, "c": c̄})``
    with W̄ in the reference's (2·n1 × n2) index order, summed over the columns of this batch."""
    d, D, N, ldx, ldyb = _layer_vjp(t, x, ybar, ljbar, _lib.COUPLING_AFFINE, "coupling_vjp")
    n1, n2 = d.n0, d.n1
    xbar = colmajor_empty(D, N, x.device)
    Wbar = torch.empty((n2, 2 * n1), dtype=torch.float32, device=x.device)  # column-major (2n1 × n2)
    cbar = torch.empty((2 * n1,), dtype=torch.float32, device=x.device)
    L_ = lib()
    ws_bytes = L_.b2b_coupling_affine_vjp_workspace_bytes(n1, n2)
    if ws_bytes == 0:
        raise B2BError(_lib.B2B_EUNSUPPORTED, "coupling_vjp: n1, n2 <= 128")
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device)
    arr = (LayerDesc * 1)(d)
    check(L_.b2b_coupling_affine_vjp_f32(arr, x.data_ptr(), ybar.data_ptr(), ljbar.data_ptr() if ljbar is not None else None,
                                         xbar.data_ptr(), Wbar.data_ptr(), cbar.data_ptr(), D, N, ldx, ldyb,
                                         _batch_view(xbar)[2], ws.data_ptr(), ws_bytes, _stream()), "b2b_coupling_affine_vjp_f32")
    return xbar, {"W": Wbar.t(), "c": cbar}


def batchnorm_vjp(t, x: torch.Tensor, ybar: torch.Tensor, ljbar: Optional[torch.Tensor] = None):
    """Vector-Jacobian product of ``with_logabsdet_jacobian(t, x)`` for ONE eval-mode InvertibleBatchNorm ``t`` (or its
    inverse): b2b_batchnorm_eval_vjp_f32.  Returns ``(xbar, {"b": b̄, "logs": l̄ogs})`` summed over the columns."""
    d, D, N, ldx, ldyb = _layer_vjp(t, x, ybar, ljbar, _lib.BATCHNORM, "batchnorm_vjp")
    xbar = colmajor_empty(D, N, x.device)
    bbar = torch.empty((D,), dtype=torch.float32, device=x.device)
    lbar = torch.empty((D,), dtype=torch.float32, device=x.device)
    L_ = lib()
    ws_bytes = L_.b2b_batchnorm_eval_vjp_workspace_bytes(D)
    if ws_bytes == 0:
        raise B2BError(_lib.B2B_EUNSUPPORTED, "batchnorm_vjp: D <= 1024")
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device)
    arr = (LayerDesc * 1)(d)
    check(L_.b2b_batchnorm_eval_vjp_f32(arr, x.data_ptr(), ybar.data_ptr(), ljbar.data_ptr() if ljbar is not None else None,
                                        xbar.data_ptr(), bbar.data_ptr(), lbar.data_ptr(), D, N, ldx, ldyb,
                                        _batch_view(xbar)[2], ws.data_ptr(), ws_bytes, _stream()), "b2b_batchnorm_eval_vjp_f32")
    return xbar, {"b": bbar, "logs": lbar}


def rqs_vjp(t, x: torch.Tensor, ybar: torch.Tensor, ljbar: Optional[torch.Tensor] = None):
    """Vector-Jacobian product of ``with_logabsdet_jacobian(t, x)`` for ONE RationalQuadraticSpline ``t`` (or its inverse,
    with ``x`` the observed batch): b2b_rqs_vjp_f32.  Returns ``(xbar, {"widths": W̄, "heights": H̄, "derivatives": D̄})``,
    the cotangents of the processed (D × K+1) knot arrays, summed over the columns of this batch."""
    d, D, N, ldx, ldyb = _layer_vjp(t, x, ybar, ljbar, _lib.RQS, "rqs_vjp")
    K1 = d.n0
    xbar = colmajor_empty(D, N, x.device)
    bars = [torch.empty((K1, D), dtype=torch.float32, device=x.device) for _ in range(3)]  # column-major (D × K1)
    L_ = lib()
    ws_bytes = L_.b2b_rqs_vjp_workspace_bytes(K1, D)
    if ws_bytes == 0:
        raise B2BError(_lib.B2B_EUNSUPPORTED, "rqs_vjp: K+1 <= 64 knots, D <= 256")
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device)
    arr = (LayerDesc * 1)(d)
    check(L_.b2b_rqs_vjp_f32(arr, x.data_ptr(), ybar.data_ptr(), ljbar.data_ptr() if ljbar is not None else None,
                             xbar.data_ptr(), bars[0].data_ptr(), bars[1].data_ptr(), bars[2].data_ptr(), D, N, ldx, ldyb,
                             _batch_view(xbar)[2], ws.data_ptr(), ws_bytes, _stream()), "b2b_rqs_vjp_f32")
    return xbar, {"widths": bars[0].t(), "heights": bars[1].t(), "derivatives": bars[2].t()}


def isinvertible(t) -> bool:
    return isinstance(t, Transform)


def isclosedform(t) -> bool:
    """isclosedform (src/interface.jl:233; planar_layer.jl:188: Inverse{PlanarLayer} is not)."""
    from .layers import PlanarLayer

    if isinstance(t, Inverse) and isinstance(t.orig, PlanarLayer):
        return False
    if isinstance(t, (ComposedFunction, Composed)):
        return all(isclosedform(b) for b in flatten(t))
    return True
