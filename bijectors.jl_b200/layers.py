"""Flow layers of the hot path: parameter structs with the reference's field names whose evaluation is a
launch of the matching libb2b.so kernel (include/b2b.h).  No arithmetic on the batch happens here.

  PlanarLayer{w,u,b}                 src/bijectors/planar_layer.jl:13-18
  RadialLayer{α_,β,z_0}              src/bijectors/radial_layer.jl:11-17
  RationalQuadraticSpline            src/bijectors/rational_quadratic_spline.jl:75-123
  PartitionMask / Coupling           src/bijectors/coupling.jl:51-118,178-259
  InvertibleBatchNorm                src/bijectors/normalise.jl:9-37
  Permute                            src/bijectors/permute.jl:84-157
  Stacked / elementwise / Shift / Scale   src/bijectors/stacked.jl, exp_log.jl, shift.jl, scale.jl
  LowerTriangular / UpperTriangular / UnitLowerTriangular / UnitUpperTriangular   LinearAlgebra's wrappers, for Scale(T)
  LULinear                           Permute(p) ∘ Scale(UnitLowerTriangular(F)) ∘ Scale(UpperTriangular(F)) as one layer
  MaskedAutoregressive               MAF / IAF's affine layer with a MADE conditioner
  LeakyReLU                          src/bijectors/leaky_relu.jl
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import B2BError, LayerDesc, LayerDesc64
from .interface import Bijector, Inverse, Transform


def _dev_f32(v, device, dtype=torch.float32) -> torch.Tensor:
    """Parameter tensor on `device`: Float32 (the hot path) or Float64 (the reference's own test precision; evaluated by
    b2b_chain_run_f64)."""
    if dtype not in (torch.float32, torch.float64):
        raise TypeError(f"parameters are Float32 or Float64, got {dtype}")
    if isinstance(v, torch.Tensor):
        t = v.detach()
    else:
        t = torch.as_tensor(np.asarray(v, dtype=np.float64 if dtype == torch.float64 else np.float32))
    t = t.to(device=device, dtype=dtype)
    return t.reshape(-1).contiguous() if t.dim() <= 1 else t.contiguous()


def _check_dtype(param: torch.Tensor, dtype, what: str) -> None:
    if param.dtype != dtype:
        raise TypeError(f"{what} has {param.dtype} parameters but the batch is {dtype}; construct the layer with dtype={dtype} "
                        "(Float32 is the hot path, Float64 the reference's test precision)")


def _dev_i32(v, device) -> torch.Tensor:
    return torch.as_tensor(np.asarray(v, dtype=np.int32)).to(device).contiguous()


def _desc(kind, inverse=False, **kw):
    """b2b_layer_desc, or b2b_layer_desc_f64 when the layer's parameters are Float64 tensors."""
    f64 = any(isinstance(v, torch.Tensor) and v.dtype == torch.float64 for v in kw.values()) or kw.pop("_f64", False)
    d = LayerDesc64() if f64 else LayerDesc()
    d.kind = kind
    d.inverse = 1 if inverse else 0
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            v = v.data_ptr()
        setattr(d, k, v)
    return d


class _ParamLayer(Bijector):
    """Common plumbing: parameters are float32 tensors on one device (`fmap`-style movement with .to())."""

    _fields: Tuple[str, ...] = ()

    def params(self) -> Dict[str, torch.Tensor]:
        """Functors.@functor analogue: the numerical parameters by reference field name."""
        return {k: getattr(self, k) for k in self._fields}

    def to(self, device):
        new = object.__new__(type(self))
        new.__dict__.update(self.__dict__)
        for k in self._fields:
            setattr(new, k, getattr(self, k).to(device))
        new._cache = {}
        return new

    @property
    def device(self):
        return getattr(self, self._fields[0]).device

    def _keepalive(self):
        return tuple(getattr(self, k) for k in self._fields)

    def __eq__(self, other):
        return type(self) is type(other) and all(
            torch.equal(getattr(self, k).cpu(), getattr(other, k).cpu()) for k in self._fields
        )

    __hash__ = object.__hash__


# --------------------------------------------------------------------------------------------------
class PlanarLayer(_ParamLayer):
    """f(z) = z + û·tanh(wᵀz + b)  (planar_layer.jl:73-80); logjac = log1p(wᵀû·sech²(wᵀz+b)) (:102-110).
    Inverse via find_alpha (:112-127,:160-185).  `b` may be a scalar or a 1-vector (first(b), :75)."""

    _fields = ("w", "u", "b")

    def __init__(self, w, u=None, b=None, device="cuda", generator: Optional[torch.Generator] = None, dtype=torch.float32):
        if isinstance(w, int):  # PlanarLayer(dims) : randn parameters (:23-28)
            dims = w
            w = torch.randn(dims, generator=generator)
            u = torch.randn(dims, generator=generator)
            b = torch.randn(1, generator=generator)
        self.w = _dev_f32(w, device, dtype)
        self.u = _dev_f32(u, device, dtype)
        self.b = _dev_f32(b, device, dtype)
        if self.w.numel() != self.u.numel():
            raise ValueError("w and u must have the same length")

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != self.w.numel():
            raise ValueError(f"DimensionMismatch: PlanarLayer has {self.w.numel()} dims, input has {D}")
        _check_dtype(self.w, dtype, "PlanarLayer")
        d = _desc(_lib.PLANAR, inverse, p0=self.w, p1=self.u, p2=self.b)
        if not self.w.is_cuda:
            # host-resident parameters (the reference's own residency: plain Arrays, planar_layer.jl:13-18):
            # run_chain routes all-planar host-parameter chains to b2b_planar_chain_hostparams_f32
            d._host_planar = (self.w, self.u, self.b)
        return [d]


class RadialLayer(_ParamLayer):
    """f(z) = z + β̂/(α+r)·(z − z₀)  (radial_layer.jl:43-53,58-72); closed-form inverse (:88-102,:124-129)."""

    _fields = ("α_", "β", "z_0")

    def __init__(self, α_, β=None, z_0=None, device="cuda", generator: Optional[torch.Generator] = None, dtype=torch.float32):
        if isinstance(α_, int) and β is None:  # RadialLayer(dims) (:22-27)
            dims = α_
            α_ = torch.randn(1, generator=generator)
            β = torch.randn(1, generator=generator)
            z_0 = torch.randn(dims, generator=generator)
        setattr(self, "α_", _dev_f32(α_, device, dtype))
        setattr(self, "β", _dev_f32(β, device, dtype))
        self.z_0 = _dev_f32(z_0, device, dtype)

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != self.z_0.numel():
            raise ValueError(f"DimensionMismatch: RadialLayer has {self.z_0.numel()} dims, input has {D}")
        _check_dtype(self.z_0, dtype, "RadialLayer")
        return [_desc(_lib.RADIAL, inverse, p0=getattr(self, "α_"), p1=getattr(self, "β"), p2=self.z_0)]


class RationalQuadraticSpline(_ParamLayer):
    """Neural-spline-flow element-wise bijector on [-B, B]^D.

    RationalQuadraticSpline(widths, heights, derivatives)     processed knots, (D × K+1) each  (:75-97)
    RationalQuadraticSpline(widths, heights, derivatives, B)  raw parameters (D×K, D×K, D×(K-1)) are
        normalised on the host exactly as the reference constructor does (:109-123): softmax → cumsum →
        [-B, B] knots, softplus derivatives with unit end slopes.  (Tiny, once per construction.)
    Matrices are given with the reference's index order: row = dimension, column = knot.
    """

    _fields = ("widths", "heights", "derivatives")

    def __init__(self, widths, heights, derivatives, B=None, device="cuda", dtype=torch.float32):
        npdt = np.float64 if dtype == torch.float64 else np.float32
        w = np.asarray(widths.detach().cpu() if isinstance(widths, torch.Tensor) else widths, dtype=npdt)
        h = np.asarray(heights.detach().cpu() if isinstance(heights, torch.Tensor) else heights, dtype=npdt)
        d = np.asarray(derivatives.detach().cpu() if isinstance(derivatives, torch.Tensor) else derivatives,
                       dtype=npdt)
        if w.ndim == 1:
            w, h, d = w[None, :], h[None, :], d[None, :]
        if B is not None:
            w, h, d = _rqs_normalise(w, h, d, float(B), npdt)
        # struct asserts (:93-94)
        assert w.shape[1] == h.shape[1] == d.shape[1], "widths, heights and derivatives need the same number of knots"
        assert np.all(d > 0), "derivatives need to be positive"
        self.K1 = int(w.shape[1])
        self.D = int(w.shape[0])
        # device copies keep Julia's column-major (D × K1) memory order == knot-major [k][i]
        self.widths = _dev_f32(np.ascontiguousarray(w.T), device, dtype)
        self.heights = _dev_f32(np.ascontiguousarray(h.T), device, dtype)
        self.derivatives = _dev_f32(np.ascontiguousarray(d.T), device, dtype)

    def knots(self):
        """(widths, heights, derivatives) as (D × K+1) numpy arrays in the reference's index order."""
        return tuple(getattr(self, k).cpu().numpy().T.copy() for k in self._fields)

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != self.D:
            raise ValueError(f"DimensionMismatch: RationalQuadraticSpline has {self.D} dims, input has {D}")
        _check_dtype(self.widths, dtype, "RationalQuadraticSpline")
        return [_desc(_lib.RQS, inverse, p0=self.widths, p1=self.heights, p2=self.derivatives, n0=self.K1)]


def _rqs_normalise(w, h, d, B, f=np.float32):
    """Host restatement of the normalising constructor (rational_quadratic_spline.jl:109-123) in the parameter eltype."""

    def softmax(v):
        e = np.exp(v - v.max(axis=1, keepdims=True))
        return (e / e.sum(axis=1, keepdims=True)).astype(f)

    def softplus(v):
        v = v.astype(np.float64)
        return np.where(v > 0, v + np.log1p(np.exp(-np.abs(v))), np.log1p(np.exp(-np.abs(v)))).astype(f)

    n = w.shape[0]
    ws = np.concatenate([np.zeros((n, 1), f), softmax(w)], axis=1)
    hs = np.concatenate([np.zeros((n, 1), f), softmax(h)], axis=1)
    ds = np.concatenate([np.ones((n, 1), f), softplus(d), np.ones((n, 1), f)], axis=1)
    W = (f(2 * B) * np.cumsum(ws, axis=1, dtype=f) - f(B)).astype(f)
    H = (f(2 * B) * np.cumsum(hs, axis=1, dtype=f) - f(B)).astype(f)
    return W, H, ds


# --------------------------------------------------------------------------------------------------
class PartitionMask:
    """PartitionMask(n, indices_1, indices_2[, indices_3]) / PartitionMask(n, indices)
    (coupling.jl:51-118).  Indices are 1-BASED like the reference; the sparse 0/1 selector matrices are
    kept as index lists (partition / combine are pure index movement, bit-exact)."""

    def __init__(self, n: int, indices_1, indices_2=None, indices_3=None):
        i1 = [int(i) for i in indices_1]
        if indices_2 is None and indices_3 is None:
            i2 = [i for i in range(1, n + 1) if i not in set(i1)]  # :107-115
            i3 = []
        elif indices_3 is None:
            i2 = [int(i) for i in indices_2]
            i3 = [i for i in range(1, n + 1) if i not in set(i1) | set(i2)]  # :85-92
        elif indices_2 is None:
            i3 = [int(i) for i in indices_3]
            i2 = [i for i in range(1, n + 1) if i not in set(i1) | set(i3)]  # :94-101
        else:
            i2, i3 = [int(i) for i in indices_2], [int(i) for i in indices_3]
        allidx = i1 + i2 + i3
        if any(i < 1 or i > n for i in allidx) or len(set(allidx)) != len(allidx):
            raise ValueError("PartitionMask indices must be disjoint and within 1:n")
        self.n, self.indices_1, self.indices_2, self.indices_3 = n, i1, i2, i3

    def __eq__(self, o):
        return (self.n, self.indices_1, self.indices_2, self.indices_3) == (o.n, o.indices_1, o.indices_2, o.indices_3)


class AffineConditioner:
    """The recognised coupling law θ(x₂) = Shift(t) ∘ Scale(exp.(s)) with [s; t] = W·x₂ + c
    (Scale scale.jl:13,31; Shift shift.jl:14,21).  W is (2·n1 × n2) in the reference's index order."""

    def __init__(self, W, c=None, device="cuda", dtype=torch.float32):
        npdt = np.float64 if dtype == torch.float64 else np.float32
        Wn = np.asarray(W.detach().cpu() if isinstance(W, torch.Tensor) else W, dtype=npdt)
        if Wn.ndim != 2 or Wn.shape[0] % 2:
            raise ValueError("W must be (2*n1, n2)")
        self.n1, self.n2 = Wn.shape[0] // 2, Wn.shape[1]
        self.W = _dev_f32(np.ascontiguousarray(Wn.T), device, dtype)  # column-major (2n1 × n2)
        cn = np.zeros(Wn.shape[0], npdt) if c is None else np.asarray(
            c.detach().cpu() if isinstance(c, torch.Tensor) else c, dtype=npdt)
        self.c = _dev_f32(cn, device, dtype)

    def to(self, device):
        new = object.__new__(AffineConditioner)
        new.n1, new.n2 = self.n1, self.n2
        new.W, new.c = self.W.to(device), self.c.to(device)
        return new

    def _tensors(self):
        return (self.W, self.c)


def _host32(v):
    return np.asarray(v.detach().cpu() if isinstance(v, torch.Tensor) else v, dtype=np.float32)


def _spline_law(who, Wn, K, B, cols):
    """(K, B, n1) of a spline conditioner whose last layer Wn has (3K−1)·n1 rows and ``cols`` columns."""
    K = int(K)
    if K < 1:
        raise ValueError(f"{who}: K must be >= 1")
    if not float(B) > 0:
        raise ValueError(f"{who}: B must be > 0")
    J = 3 * K - 1
    if Wn.ndim != 2 or Wn.shape[0] == 0 or Wn.shape[0] % J:
        raise ValueError(f"{who}: W must be ((3K-1)*n1, {cols}) = ({J}*n1, {cols}), got {Wn.shape}")
    return K, float(B), Wn.shape[0] // J


def _bias(c, name, n, device):
    if c is None:
        return None
    cn = _host32(c).reshape(-1)
    if cn.shape != (n,):
        raise ValueError(f"{name} must have {n} entries, got {cn.shape}")
    return _dev_f32(cn, device)


_ACT = {"tanh": _lib.ACT_TANH, "leaky_relu": _lib.ACT_LEAKY_RELU}


class SplineConditioner:
    """The neural-spline coupling law (Durkan et al. 2019) θ(x₂) = RationalQuadraticSpline(reshape(v[1:n1K], n1, K),
    reshape(v[n1K+1:2n1K], n1, K), reshape(v[2n1K+1:end], n1, K−1), B) with v = W·x₂ + c -- the reference's own
    constructor (rational_quadratic_spline.jl:109-123) applied to a linear conditioner.  W is ((3K−1)·n1 × n2) in the
    reference's index order (row i + n1·k of v is row i, bin k of its block); c has (3K−1)·n1 entries (None = no shift,
    the descriptor's c is NULL).  Float32 only.  Runs as B2B_COUPLING_RQS: n1, n2 <= 128, 2 <= K <= 16, D <= 1024."""

    def __init__(self, W, c=None, *, K: int, B: float, device="cuda", dtype=torch.float32):
        if dtype != torch.float32:
            raise TypeError("SplineConditioner: the spline coupling layer runs in Float32 only")
        Wn = _host32(W)
        self.K, self.B, self.n1 = _spline_law("SplineConditioner", Wn, K, B, "n2")
        self.n2 = Wn.shape[1]
        self.W = _dev_f32(np.ascontiguousarray(Wn.T), device)  # column-major ((3K−1)n1 × n2)
        self.c = _bias(c, "c", Wn.shape[0], device)

    def to(self, device):
        new = object.__new__(SplineConditioner)
        new.__dict__.update(self.__dict__)
        new.W = self.W.to(device)
        new.c = None if self.c is None else self.c.to(device)
        return new

    def _tensors(self):
        return (self.W, self.c)


class _NetworkConditioner:
    """A conditioner whose parameters come from a hidden layer h = σ.(W₁·x₂ + c₁) and a last layer W₂·h + c₂."""

    _ACT = _ACT
    _fields = ("W1", "c1", "W2", "c2")  # the device tensors, in the order of the descriptor's p0 .. p3

    def _network(self, who, activation, slope, dtype):
        """Checks the element type and the activation and sets activation and slope."""
        if dtype != torch.float32:
            raise TypeError(f"{who}: the network coupling layers run in Float32 only")
        if activation not in _ACT:
            raise ValueError(f"{who}: activation must be one of {sorted(_ACT)}, got {activation!r}")
        self.activation, self.slope = activation, float(slope)

    def _first_layer(self, name, W):
        """Checks the input layer (H × n2), sets H and n2 and returns it column-major on the host."""
        Wn = _host32(W)
        if Wn.ndim != 2 or Wn.shape[0] == 0:
            raise ValueError(f"{name} must be (H, n2), got {Wn.shape}")
        self.H, self.n2 = Wn.shape
        return np.ascontiguousarray(Wn.T)

    def _hidden_layer(self, who, W1, c1, activation, slope, dtype, device):
        """Checks the hidden layer and sets activation, slope, H, n2, W1 (column-major) and c1 (None: NULL pointer)."""
        self._network(who, activation, slope, dtype)
        self.W1 = _dev_f32(self._first_layer("W1", W1), device)  # column-major (H × n2)
        self.c1 = _bias(c1, "c1", self.H, device)

    def to(self, device):
        new = object.__new__(type(self))
        new.__dict__.update(self.__dict__)
        for k in self._fields:
            t = getattr(self, k)
            setattr(new, k, None if t is None else t.to(device))
        return new

    def _tensors(self):
        return tuple(getattr(self, k) for k in self._fields)


class MLPConditioner(_NetworkConditioner):
    """The neural-network coupling law of RealNVP: θ(x₂) = Shift(t) ∘ Scale(exp.(s)) with
    [s; t] = W₂·σ.(W₁·x₂ + c₁) + c₂, one hidden layer of width H and σ = tanh or LeakyReLU(slope) (slope 0 is ReLU;
    v >= 0 ? v : slope·v, leaky_relu.jl:18-29).  W1 is (H × n2) and W2 (2·n1 × H) in the reference's index order, rows
    1..n1 of W2 giving s and the rest t as for :class:`AffineConditioner`; c1 (H) and c2 (2·n1) may be None (no shift,
    the descriptor's pointer is NULL).  Float32 only.  Runs as B2B_COUPLING_MLP: n1, n2 <= 128, H <= 256, D <= 1024."""

    def __init__(self, W1, c1, W2, c2, activation="tanh", slope=0.0, device="cuda", dtype=torch.float32):
        self._hidden_layer("MLPConditioner", W1, c1, activation, slope, dtype, device)
        W2n = _host32(W2)
        if W2n.ndim != 2 or W2n.shape[0] == 0 or W2n.shape[0] % 2 or W2n.shape[1] != self.H:
            raise ValueError(f"W2 must be (2*n1, H) with H = {self.H}, got {W2n.shape}")
        self.n1 = W2n.shape[0] // 2
        self.W2 = _dev_f32(np.ascontiguousarray(W2n.T), device)  # column-major (2n1 × H)
        self.c2 = _bias(c2, "c2", 2 * self.n1, device)


class MLPSplineConditioner(_NetworkConditioner):
    """The neural spline flow's coupling law (Durkan et al. 2019): θ(x₂) = RationalQuadraticSpline(…, B) as for
    :class:`SplineConditioner`, with the raw knots v = W₂·σ.(W₁·x₂ + c₁) + c₂ from one hidden layer of width H as for
    :class:`MLPConditioner`.  W1 is (H × n2) and W2 ((3K−1)·n1 × H) in the reference's index order; c1 (H) and c2
    ((3K−1)·n1) may be None.  Float32 only.  Runs as B2B_COUPLING_MLP_RQS: n1, n2 <= 128, H <= 128, 2 <= K <= 16,
    D <= 1024."""

    def __init__(self, W1, c1, W2, c2, *, K: int, B: float, activation="tanh", slope=0.0, device="cuda",
                 dtype=torch.float32):
        self._hidden_layer("MLPSplineConditioner", W1, c1, activation, slope, dtype, device)
        W2n = _host32(W2)
        self.K, self.B, self.n1 = _spline_law("MLPSplineConditioner", W2n, K, B, "H")
        if W2n.shape[1] != self.H:
            raise ValueError(f"W2 must be ((3K-1)*n1, H) with H = {self.H}, got {W2n.shape}")
        self.W2 = _dev_f32(np.ascontiguousarray(W2n.T), device)  # column-major ((3K−1)n1 × H)
        self.c2 = _bias(c2, "c2", W2n.shape[0], device)


class _DeepNetworkConditioner(_NetworkConditioner):
    """A conditioner whose parameters come from M >= 2 hidden layers h_1 = σ.(W_in·x₂ + c_1),
    h_l = σ.(W_l·h_{l−1} + c_l) (l = 2..M) and a last layer W_out·h_M + c_out.  Device tensors: W_in, W_hid (M−1, H, H:
    each matrix column-major, back to back), W_out and c (every bias packed); ``weights`` / ``biases`` give per-layer
    views in the reference's orientation."""

    _fields = ("W_in", "W_hid", "W_out", "c")
    _shallow = ""  # the one-hidden-layer conditioner of the same law

    def _deep_network(self, who, weights, biases, activation, slope, dtype, device, last_layer):
        """Checks the layers and sets activation, slope, M, H, n2, W_in, W_hid, W_out and c; ``last_layer(W_out)``
        checks the law's last layer (rows × H) and sets n1."""
        self._network(who, activation, slope, dtype)
        weights = list(weights)
        if len(weights) < 3:
            raise ValueError(f"{who}: weights must be [W_in, W_2, …, W_M, W_out] with M >= 2 hidden layers "
                             f"(one hidden layer is {self._shallow}), got {len(weights)} matrices")
        self.M = len(weights) - 1
        W_in = self._first_layer("W_in", weights[0])
        H = self.H
        hid = [_host32(W) for W in weights[1:-1]]
        for l, W in enumerate(hid, start=2):
            if W.shape != (H, H):
                raise ValueError(f"W_{l} must be (H, H) with H = {H}, got {W.shape}")
        W_out = _host32(weights[-1])
        last_layer(W_out)
        self.W_in = _dev_f32(W_in, device)  # column-major (H × n2)
        self.W_hid = _dev_f32(np.ascontiguousarray(np.stack([W.T for W in hid])), device)  # [l − 2] = W_l column-major
        self.W_out = _dev_f32(np.ascontiguousarray(W_out.T), device)  # column-major (rows × H)
        self.c = None
        if biases is not None:
            biases = list(biases)
            if len(biases) != self.M + 1:
                raise ValueError(f"biases must be None or all {self.M + 1} vectors [c_1, …, c_{self.M}, c_out], "
                                 f"got {len(biases)}")
            names = [f"c_{l}" for l in range(1, self.M + 1)] + ["c_out"]
            sizes = [H] * self.M + [W_out.shape[0]]
            parts = [_host32(b).reshape(-1) for b in biases]
            for name, n, b in zip(names, sizes, parts):
                if b.shape != (n,):
                    raise ValueError(f"{name} must have {n} entries, got {b.shape}")
            self.c = _dev_f32(np.concatenate(parts), device)

    @property
    def weights(self):
        """[W_in, W_2, …, W_M, W_out] as views of the device tensors, in the reference's orientation."""
        return [self.W_in.t()] + [W.t() for W in self.W_hid] + [self.W_out.t()]

    @property
    def biases(self):
        """[c_1, …, c_M, c_out] as views of the packed bias, or None."""
        if self.c is None:
            return None
        H, M = self.H, self.M
        return [self.c[l * H:(l + 1) * H] for l in range(M)] + [self.c[M * H:]]


class DeepMLPConditioner(_DeepNetworkConditioner):
    """The RealNVP coupling law θ(x₂) = Shift(t) ∘ Scale(exp.(s)) of :class:`MLPConditioner` with a deeper network, a
    Flux ``Chain(Dense(n2, H, σ), Dense(H, H, σ), …, Dense(H, 2n1))``: h_1 = σ.(W_in·x₂ + c_1), h_l = σ.(W_l·h_{l−1} + c_l)
    for l = 2..M, [s; t] = W_out·h_M + c_out.  ``weights = [W_in (H × n2), W_2 … W_M (H × H), W_out (2·n1 × H)]`` in the
    reference's index order, M >= 2 hidden layers, rows 1..n1 of W_out giving s.  ``biases`` is None (no biases at all,
    the descriptor's pointer is NULL) or all M + 1 vectors ``[c_1 … c_M (H each), c_out (2·n1)]``, so that training never
    adds a bias the network did not have.  Float32 only.  Runs as B2B_COUPLING_DEEP_MLP: n1, n2 <= 128, H <= 128,
    M <= 4, D <= 1024.  Device tensors: W_in, W_hid (M−1, H, H: each matrix column-major, back to back), W_out and c
    (every bias packed); ``weights`` / ``biases`` give per-layer views in the reference's orientation."""

    _shallow = "MLPConditioner"

    def __init__(self, weights, biases=None, *, activation="tanh", slope=0.0, device="cuda", dtype=torch.float32):
        self._deep_network("DeepMLPConditioner", weights, biases, activation, slope, dtype, device, self._affine_out)

    def _affine_out(self, W_out):
        if W_out.ndim != 2 or W_out.shape[0] == 0 or W_out.shape[0] % 2 or W_out.shape[1] != self.H:
            raise ValueError(f"W_out must be (2*n1, H) with H = {self.H}, got {W_out.shape}")
        self.n1 = W_out.shape[0] // 2


class DeepMLPSplineConditioner(_DeepNetworkConditioner):
    """The neural spline flow's coupling law (Durkan et al. 2019) with a deep network: θ(x₂) =
    RationalQuadraticSpline(…, B) as for :class:`SplineConditioner`, with the raw knots v = W_out·h_M + c_out from the M
    hidden layers of :class:`DeepMLPConditioner`, a Flux ``Chain(Dense(n2, H, σ), Dense(H, H, σ), …,
    Dense(H, (3K−1)·n1))``.  ``weights = [W_in (H × n2), W_2 … W_M (H × H), W_out ((3K−1)·n1 × H)]`` in the reference's
    index order, M >= 2 hidden layers; ``biases`` is None or all M + 1 vectors ``[c_1 … c_M (H each),
    c_out ((3K−1)·n1)]``.  Float32 only.  Runs as B2B_COUPLING_DEEP_MLP_RQS: n1, n2 <= 128, H <= 128, 2 <= K <= 16,
    M <= 4, D <= 1024.  Device tensors and views as for :class:`DeepMLPConditioner`."""

    _shallow = "MLPSplineConditioner"

    def __init__(self, weights, biases=None, *, K: int, B: float, activation="tanh", slope=0.0, device="cuda",
                 dtype=torch.float32):
        def spline_out(W_out):
            self.K, self.B, self.n1 = _spline_law("DeepMLPSplineConditioner", W_out, K, B, "H")
            if W_out.shape[1] != self.H:
                raise ValueError(f"W_out must be ((3K-1)*n1, H) with H = {self.H}, got {W_out.shape}")

        self._deep_network("DeepMLPSplineConditioner", weights, biases, activation, slope, dtype, device, spline_out)


class Coupling(_ParamLayer):
    """Coupling(θ, mask) (coupling.jl:178-181).  θ is an arbitrary closure in the reference; the device
    path supports the recognised :class:`AffineConditioner`, :class:`SplineConditioner`, :class:`MLPConditioner`,
    :class:`MLPSplineConditioner`, :class:`DeepMLPConditioner` and :class:`DeepMLPSplineConditioner` and raises for
    anything else (no CPU fallback)."""

    _fields = ()

    def __init__(self, θ, mask, device="cuda"):
        if isinstance(mask, int):  # Coupling(θ, n): first n÷2 rows transformed (:183-186)
            mask = PartitionMask(mask, range(1, mask // 2 + 1))
        if not isinstance(θ, (AffineConditioner, SplineConditioner, MLPConditioner, MLPSplineConditioner,
                              DeepMLPConditioner, DeepMLPSplineConditioner)):
            raise B2BError(_lib.B2B_EUNSUPPORTED, "Coupling: only AffineConditioner, SplineConditioner, MLPConditioner, "
                                                  "MLPSplineConditioner, DeepMLPConditioner and DeepMLPSplineConditioner "
                                                  "laws run on the device path")
        if θ.n1 != len(mask.indices_1) or θ.n2 != len(mask.indices_2):
            raise ValueError("conditioner shape does not match the PartitionMask")
        self.θ, self.mask = θ, mask
        self._idx1 = _dev_i32(np.asarray(mask.indices_1) - 1, self.device)
        self._idx2 = _dev_i32(np.asarray(mask.indices_2) - 1, self.device)

        def first_row(idx):  # 0-based first row when the list is a contiguous increasing range, else -1
            a = np.asarray(idx)
            return int(a[0] - 1) if len(a) and np.array_equal(a, np.arange(a[0], a[0] + len(a))) else -1

        self._row1, self._row2 = first_row(mask.indices_1), first_row(mask.indices_2)

    @property
    def device(self):
        return self.θ._tensors()[0].device

    def to(self, device):
        """fmap-style movement: the conditioner's tensors AND the index lists follow."""
        return Coupling(self.θ.to(device), self.mask)

    def _keepalive(self):
        return self.θ._tensors() + (self._idx1, self._idx2)

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != self.mask.n:
            raise ValueError(f"DimensionMismatch: Coupling mask has {self.mask.n} dims, input has {D}")
        _check_dtype(self.θ._tensors()[0], dtype, "Coupling")
        if isinstance(self.θ, MLPConditioner):
            θ = self.θ
            return [_desc(_lib.COUPLING_MLP, inverse, p0=θ.W1, p1=θ.c1 if θ.c1 is not None else 0, p2=θ.W2,
                          p3=θ.c2 if θ.c2 is not None else 0, i0=self._idx1, i1=self._idx2, n0=θ.n1, n1=θ.n2, n2=θ.H,
                          n3=θ._ACT[θ.activation], f0=θ.slope)]
        if isinstance(self.θ, DeepMLPConditioner):
            θ = self.θ
            return [_desc(_lib.COUPLING_DEEP_MLP, inverse, p0=θ.W_in, p1=θ.W_hid, p2=θ.W_out,
                          p3=θ.c if θ.c is not None else 0, i0=self._idx1, i1=self._idx2, n0=θ.n1, n1=θ.n2, n2=θ.H,
                          n3=θ._ACT[θ.activation] | (θ.M << 8), f0=θ.slope)]
        if isinstance(self.θ, DeepMLPSplineConditioner):
            θ = self.θ
            return [_desc(_lib.COUPLING_DEEP_MLP_RQS, inverse, p0=θ.W_in, p1=θ.W_hid, p2=θ.W_out,
                          p3=θ.c if θ.c is not None else 0, i0=self._idx1, i1=self._idx2, n0=θ.n1, n1=θ.n2, n2=θ.H,
                          n3=θ._ACT[θ.activation] | (θ.K << 8) | (θ.M << 16), f0=θ.slope, f1=θ.B)]
        if isinstance(self.θ, MLPSplineConditioner):
            θ = self.θ
            return [_desc(_lib.COUPLING_MLP_RQS, inverse, p0=θ.W1, p1=θ.c1 if θ.c1 is not None else 0, p2=θ.W2,
                          p3=θ.c2 if θ.c2 is not None else 0, i0=self._idx1, i1=self._idx2, n0=θ.n1, n1=θ.n2, n2=θ.H,
                          n3=θ._ACT[θ.activation] | (θ.K << 8), f0=θ.slope, f1=θ.B)]
        if isinstance(self.θ, SplineConditioner):
            return [_desc(_lib.COUPLING_RQS, inverse, p0=self.θ.W, p1=self.θ.c if self.θ.c is not None else 0,
                          i0=self._idx1, i1=self._idx2, n0=self.θ.n1, n1=self.θ.n2, n2=self.θ.K, n3=0, f0=self.θ.B)]
        return [_desc(_lib.COUPLING_AFFINE, inverse, p0=self.θ.W, p1=self.θ.c, i0=self._idx1, i1=self._idx2,
                      n0=self.θ.n1, n1=self.θ.n2, n2=self._row1, n3=self._row2)]

    def __eq__(self, o):
        if not (isinstance(o, Coupling) and type(self.θ) is type(o.θ) and self.mask == o.mask):
            return False
        if isinstance(self.θ, SplineConditioner) and (self.θ.K, self.θ.B) != (o.θ.K, o.θ.B):
            return False
        if isinstance(self.θ, (MLPSplineConditioner, DeepMLPSplineConditioner)) and (self.θ.K, self.θ.B) != (o.θ.K, o.θ.B):
            return False
        if isinstance(self.θ, _DeepNetworkConditioner) and self.θ.M != o.θ.M:
            return False
        if isinstance(self.θ, _NetworkConditioner) and \
                (self.θ.activation, self.θ.slope) != (o.θ.activation, o.θ.slope):
            return False
        return all((a is None) == (b is None) and (a is None or torch.equal(a, b))
                   for a, b in zip(self.θ._tensors(), o.θ._tensors()))

    __hash__ = object.__hash__


def coupling(cl: Coupling):
    """coupling(cl) = cl.θ (coupling.jl:193)."""
    return cl.θ


# --------------------------------------------------------------------------------------------------
class InvertibleBatchNorm(_ParamLayer):
    """InvertibleBatchNorm(chs; eps=1f-5, mtm=1f-1) (normalise.jl:9-37); eval mode (:61-67,:74-86).
    The reference's global `istraining()` switch (:7) is the explicit `training` flag here: a training-mode layer
    computes batch statistics and updates its moving statistics in place (`train_forward`, :51-60)."""

    _fields = ("b", "logs", "m", "v")

    def __init__(self, chs=None, *, b=None, logs=None, m=None, v=None, eps=1e-5, mtm=1e-1, device="cuda",
                 training=False, dtype=torch.float32):
        if chs is not None:
            b, logs, m, v = np.zeros(chs), np.zeros(chs), np.zeros(chs), np.ones(chs)
        self.b, self.logs, self.m, self.v = (_dev_f32(t, device, dtype) for t in (b, logs, m, v))
        self.eps, self.mtm, self.training = float(np.float32(eps)), float(np.float32(mtm)), training

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != self.b.numel():
            # error text of normalise.jl:43-45
            raise RuntimeError(f"InvertibleBatchNorm expected {self.b.numel()} channels, got {D}")
        if self.training:
            raise B2BError(_lib.B2B_EUNSUPPORTED, "InvertibleBatchNorm in training mode cannot be fused into a chain "
                                                  "or inverted (normalise.jl:75); call it on its own")
        _check_dtype(self.b, dtype, "InvertibleBatchNorm")
        return [_desc(_lib.BATCHNORM, inverse, p0=self.b, p1=self.logs, p2=self.m, p3=self.v, f0=self.eps)]

    def _expanded(self, S: int):
        """The same eval-mode layer with every channel's parameters repeated S times (rows s + S·c of a (d₁⋯d_k·C)×B
        view of an array with k leading spatial axes; interface._batchnorm_nd).  Rebuilt on every call: the fields are
        trainable and may have changed."""
        out = InvertibleBatchNorm.__new__(InvertibleBatchNorm)
        out.b, out.logs, out.m, out.v = (torch.repeat_interleave(p, S) for p in (self.b, self.logs, self.m, self.v))
        out.eps, out.mtm, out.training = self.eps, self.mtm, False
        return out

    def train_forward(self, x, comm=None):
        """with_logabsdet_jacobian(bn, x) with istraining() == true (normalise.jl:51-69): batch statistics (over all
        ranks of `comm`, a distributed.Communicator, when given), in-place moving-average update of self.m / self.v,
        output and logjac from the batch statistics."""
        from .interface import _batch_view, _stream, colmajor_empty
        from ._lib import check, lib

        D, N, ldx = _batch_view(x)
        if D != self.b.numel():
            raise RuntimeError(f"InvertibleBatchNorm expected {self.b.numel()} channels, got {D}")
        y = colmajor_empty(D, N, x.device)
        lj = torch.empty((N,), dtype=torch.float32, device=x.device)
        nbytes = lib().b2b_batchnorm_train_workspace_bytes(D)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=x.device)
        handle = comm.handle if (comm is not None and getattr(comm, "handle", None) is not None) else None
        check(lib().b2b_batchnorm_train_fwd_f32(x.data_ptr(), y.data_ptr(), lj.data_ptr(), self.b.data_ptr(),
                                                self.logs.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.eps,
                                                self.mtm, D, N, ldx, D, 0, handle, ws.data_ptr(), nbytes, _stream()),
              "b2b_batchnorm_train_fwd_f32")
        return y, lj


# --------------------------------------------------------------------------------------------------
class Permute(_ParamLayer):
    """Permute(indices) / Permute(n, src=>dst...) / Permute(n, [srcs]=>[dsts]...) / Permute(A)
    (permute.jl:84-150).  1-based like the reference.  transform = A*x as index movement (:152),
    batched logjac = zeros(N) (:155)."""

    _fields = ()

    def __init__(self, *args, device="cuda"):
        if len(args) == 1 and np.ndim(args[0]) == 1:
            dst = self._from_indices(list(args[0]))
        elif len(args) == 1 and np.ndim(args[0]) == 2:
            dst = self._from_matrix(np.asarray(args[0]))
        else:
            dst = self._from_pairs(int(args[0]), args[1:])
        self.dst_of_src = dst  # 0-based numpy: y[dst[i]] = x[i]
        self._dst = _dev_i32(dst, device)

    @staticmethod
    def _from_indices(indices):
        n = len(indices)
        if sorted(indices) != list(range(1, n + 1)):
            raise ValueError("ArgumentError: indices is not a permutation of 1:n")
        return np.asarray(indices, dtype=np.int64) - 1  # A[idx, i] = 1  (:95-97)

    @staticmethod
    def _from_matrix(A):
        if A.shape[0] != A.shape[1] or not (np.all((A == 0) | (A == 1)) and np.all(A.sum(0) == 1) and np.all(A.sum(1) == 1)):
            raise ValueError("ArgumentError: not a permutation matrix")
        return np.argmax(A, axis=0).astype(np.int64)

    @staticmethod
    def _from_pairs(n, pairs):
        dst = np.arange(n, dtype=np.int64)
        dests, sources = set(), set()
        for src, d in pairs:
            srcs = list(src) if np.ndim(src) else [src]
            dsts = list(d) if np.ndim(d) else [d]
            if len(srcs) != len(dsts):
                raise ValueError(f"ArgumentError: {srcs} => {dsts} is not bijective")  # :132
            for s_, d_ in zip(srcs, dsts):
                if d_ in dests:
                    raise ValueError(f"ArgumentError: {d_} used more than once")
                if s_ in sources:
                    raise ValueError(f"ArgumentError: {s_} used more than once")
                dests.add(d_)
                sources.add(s_)
                dst[s_ - 1] = d_ - 1
        if (sources & dests) != (sources | dests):  # :119,:145
            raise ValueError(f"ArgumentError: {sources} ∩ {dests} ≠ {sources} ∪ {dests}")
        return dst

    @property
    def A(self):
        n = len(self.dst_of_src)
        A = np.zeros((n, n))
        A[self.dst_of_src, np.arange(n)] = 1.0
        return A

    @property
    def device(self):
        return self._dst.device

    def to(self, device):
        new = object.__new__(Permute)
        new.dst_of_src = self.dst_of_src
        new._dst = self._dst.to(device)
        return new

    def _keepalive(self):
        return (self._dst,)

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != len(self.dst_of_src):
            raise ValueError(f"DimensionMismatch: Permute has {len(self.dst_of_src)} dims, input has {D}")
        return [_desc(_lib.PERMUTE, inverse, i0=self._dst, _f64=dtype == torch.float64)]

    def __eq__(self, o):
        return isinstance(o, Permute) and np.array_equal(self.dst_of_src, o.dst_of_src)

    __hash__ = object.__hash__


# --------------------------------------------------------------------------------------------------
class Elementwise(Bijector):
    """elementwise(f) = Base.Fix1(broadcast, f) (interface.jl:33) for f ∈ {exp, log, identity}.

    On a HOST vector (BASELINE config 1: Float64, length 1024 -- API plumbing, not the hot path) it returns
    (f.(x), Σ logjac) with the reference's scalar-sum semantics (exp_log.jl:6,9).  Inside Stacked, and on
    device batches, rows are evaluated by the stacked_elementwise kernel with a per-COLUMN logjac."""

    def __init__(self, f: str):
        if f not in ("exp", "log", "identity"):
            raise B2BError(_lib.B2B_EUNSUPPORTED, f"elementwise({f})")
        self.f = f

    code = property(lambda s: {"exp": _lib.EW_EXP, "log": _lib.EW_LOG, "identity": _lib.EW_IDENTITY}[s.f])
    a = 0.0

    def _inverse(self):
        return Elementwise({"exp": "log", "log": "exp", "identity": "identity"}[self.f])

    def _host_wladj(self, x):
        xt = torch.as_tensor(x)
        if self.f == "exp":
            return torch.exp(xt), xt.sum()
        if self.f == "log":
            return torch.log(xt), -torch.log(xt).sum()
        return xt, xt.new_zeros(())

    def _descs(self, inverse, D, dtype=torch.float32):
        return _as_stacked(self, D, dtype)._descs(inverse, D, dtype)

    def __eq__(self, o):
        return isinstance(o, Elementwise) and o.f == self.f

    __hash__ = object.__hash__


def elementwise(f):
    name = f if isinstance(f, str) else {math.exp: "exp", math.log: "log", np.exp: "exp", np.log: "log",
                                         torch.exp: "exp", torch.log: "log"}.get(f, getattr(f, "__name__", str(f)))
    return Elementwise(name)


def _as_stacked(b, D, dtype=torch.float32):
    """A whole-column elementwise law is a one-block Stacked; cached on the object so the device tables
    outlive the asynchronous launch."""
    cache = b.__dict__.setdefault("_stacked_cache", {})
    key = (D, dtype)
    if key not in cache:
        cache[key] = Stacked([b], [(1, D)], dtype=dtype)
    return cache[key]


class _ElementwiseLaw(Bijector):
    """Shift / Scale / LeakyReLU with a scalar parameter -- the law's row of a Stacked table (B2B_STACKED_EW), constant --
    or with a vector a[D]: the law on every row with the row's own parameter a[r], one B2B_ELEMENTWISE_VEC descriptor
    whose `a` is trainable (shift.jl, scale.jl:16,31-32, leaky_relu.jl:25-29; Optimisers.jl trains array leaves).  The
    vector lives in the device tensor ``_a`` of the `dtype` given, Float32 (the hot path) or Float64; a 1-D tensor or
    array builds it, a Python scalar or 0-d value the scalar form.  The vector form is not a Stacked block, and its
    inverse is Inverse(layer) on the same tensor, so that reverse mode reaches it."""

    code: int

    def _init_law(self, a, device, dtype):
        if (a.dim() if isinstance(a, torch.Tensor) else np.ndim(a)) == 1:
            self._a, self._s = _dev_f32(a, device, dtype), None
        else:
            self._a, self._s = None, float(a)

    @property
    def vector(self) -> bool:
        return self._a is not None

    @property
    def a(self):
        return self._a if self.vector else self._s

    @property
    def device(self):
        return self._a.device

    def to(self, device):
        if not self.vector:
            return self
        new = object.__new__(type(self))
        new.__dict__.update(self.__dict__)
        new._a = self._a.to(device)
        return new

    def _keepalive(self):
        return (self._a,) if self.vector else ()

    def _inverse(self):
        return Inverse(self) if self.vector else self._scalar_inverse()

    def _descs(self, inverse, D, dtype=torch.float32):
        if not self.vector:
            return _as_stacked(self, D, dtype)._descs(inverse, D, dtype)
        if D != self._a.numel():
            raise ValueError(f"DimensionMismatch: {type(self).__name__} has {self._a.numel()} dims, input has {D}")
        _check_dtype(self._a, dtype, type(self).__name__)
        return [_desc(_lib.ELEMENTWISE_VEC, inverse, n0=self.code, p0=self._a)]

    def __eq__(self, o):
        if type(o) is not type(self) or o.vector != self.vector:
            return False
        return torch.equal(self._a.cpu(), o._a.cpu()) if self.vector else o._s == self._s

    __hash__ = object.__hash__


class Shift(_ElementwiseLaw):
    """Shift(a): y = a .+ x, logjac 0 (shift.jl:4-24); a scalar `a` (also a Stacked block) or a trainable vector a[D]."""

    code = _lib.EW_SHIFT

    def __init__(self, a, device="cuda", dtype=torch.float32):
        self._init_law(a, device, dtype)

    def _scalar_inverse(self):
        return Shift(-self.a)  # shift.jl:12


class _Triangular:
    """LinearAlgebra's triangular view of a square matrix: only the triangle is read, and the unit forms take the diagonal
    as 1 without reading it.  `Scale` of one is the triangular layer (B2B_SCALE_TRIANGULAR); the wrapper itself only
    holds the matrix."""

    upper: bool
    unit: bool

    def __init__(self, data):
        shape = tuple(data.shape) if isinstance(data, torch.Tensor) else np.shape(data)
        if len(shape) != 2 or shape[0] != shape[1]:
            raise ValueError(f"DimensionMismatch: {type(self).__name__} needs a square matrix, got {shape}")
        self.data = data

    def __repr__(self):
        return f"{type(self).__name__}({self.data!r})"


class LowerTriangular(_Triangular):
    upper, unit = False, False


class UpperTriangular(_Triangular):
    upper, unit = True, False


class UnitLowerTriangular(_Triangular):
    upper, unit = False, True


class UnitUpperTriangular(_Triangular):
    upper, unit = True, True


class Scale(_ElementwiseLaw):
    """Scale(a): y = a .* x, logjac = log|a| per element (scale.jl:1-39) for a scalar `a` (also a Stacked block) or a
    trainable vector a[D] (scale.jl:16,31-32).

    A square matrix `a` gives the dense layer Scale{<:AbstractMatrix} (scale.jl:14,17,35-36): y = A x, inverse A \\ y,
    logjac = logabsdet(A)[1] per column, with A trainable (B2B_SCALE_MATRIX; Float32 only, D <= 256).  The device tensor
    `_A` holds A column-major, i.e. Aᵀ row-major (as MvNormal's scale_tril); `.a` returns A in the user's orientation.
    A singular A is the caller's responsibility: the forward gives logjac = −Inf, the inverse non-finite values.

    A `LowerTriangular`, `UpperTriangular`, `UnitLowerTriangular` or `UnitUpperTriangular` `a` gives the triangular layer
    (B2B_SCALE_TRIANGULAR; Float32 D <= 256 or Float64 D <= 2048): y = T x, inverse a triangular solve, logjac = Σ log|Tᵢᵢ|
    (0 for the unit forms), reading only the triangle.  `_A` holds T column-major as for the dense form, its entries
    outside the triangle as given (training never changes them: T̄ is 0 there); `.a` returns the wrapper."""

    code = _lib.EW_SCALE

    def __init__(self, a, device="cuda", dtype=torch.float32):
        self._tri = None
        if isinstance(a, _Triangular):
            T = a.data.detach() if isinstance(a.data, torch.Tensor) else torch.as_tensor(np.asarray(a.data, dtype=np.float64))
            self._A = _dev_f32(T.t(), device, dtype)
            self._tri = type(a)
            self._a = self._s = None
            return
        if (a.dim() if isinstance(a, torch.Tensor) else np.ndim(a)) == 2:
            if dtype != torch.float32:
                raise TypeError(f"a dense Scale has Float32 parameters only, got {dtype}")
            A = a.detach() if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, dtype=np.float32))
            if A.shape[0] != A.shape[1]:
                raise ValueError(f"DimensionMismatch: Scale needs a square matrix, got {tuple(A.shape)}")
            self._A = A.to(device=device, dtype=torch.float32).t().contiguous()
            self._a = self._s = None
            return
        self._A = None
        self._init_law(a, device, dtype)

    @property
    def dense(self) -> bool:
        return self._A is not None and self._tri is None

    @property
    def triangular(self) -> bool:
        return self._tri is not None

    @property
    def a(self):
        if self.triangular:
            return self._tri(self._A.t())
        return self._A.t() if self.dense else _ElementwiseLaw.a.fget(self)

    @property
    def device(self):
        return self._A.device if self._A is not None else self._a.device

    def to(self, device):
        new = object.__new__(Scale)
        new.__dict__.update(self.__dict__)
        if self._A is not None:
            new._A = self._A.to(device)
        elif self.vector:
            new._a = self._a.to(device)
        return new

    def _keepalive(self):
        return (self._A,) if self._A is not None else _ElementwiseLaw._keepalive(self)

    def _inverse(self):
        return Inverse(self)  # the scalar form included, as before: the inverse flag on the same table

    def _descs(self, inverse, D, dtype=torch.float32):
        if self._A is None:
            return _ElementwiseLaw._descs(self, inverse, D, dtype)
        if D != self._A.shape[0]:
            raise ValueError(f"DimensionMismatch: Scale has a {self._A.shape[0]} x {self._A.shape[0]} matrix, input has {D} dims")
        _check_dtype(self._A, dtype, "Scale")
        if self.triangular:
            return [_desc(_lib.SCALE_TRIANGULAR, inverse, n0=int(self._tri.upper), n1=int(self._tri.unit), p0=self._A)]
        return [_desc(_lib.SCALE_MATRIX, inverse, p0=self._A)]

    def __eq__(self, o):
        if not isinstance(o, Scale) or self.dense != o.dense or self._tri is not o._tri:
            return False
        return torch.equal(self._A.cpu(), o._A.cpu()) if self._A is not None else _ElementwiseLaw.__eq__(self, o)

    __hash__ = object.__hash__


class LULinear(_ParamLayer):
    """LULinear(F, p=None): the LU-parameterised invertible linear layer of Glow (its invertible 1×1 convolution) and of
    nflows, y = P·L·U·x, one layer for `Permute(p) ∘ Scale(UnitLowerTriangular(F)) ∘ Scale(UpperTriangular(F))`
    (B2B_SCALE_LU; Float32 D <= 256, Float64 D <= 2048).

    F packs both factors as LAPACK getrf and Julia's `lu(A).factors` do: L strictly below the diagonal (its unit diagonal
    implied, not read), U on and above it.  `p` is 1-based like `Permute(indices)` and `lu(A).p`: row r of L·U·x goes to
    row p[r] of y, so `LULinear(lu(A).factors, lu(A).p)` is y = A x; None is the identity.  logjac = Σ log|Uᵢᵢ| per column,
    and `inverse(layer)` is x = U⁻¹ L⁻¹ Pᵀ y.  F trains as one parameter, both triangles (cotangent key `factors`); p is
    fixed.  A zero Uᵢᵢ is the caller's responsibility.  `_F` holds F column-major (Fᵀ row-major), as Scale's `_A`."""

    _fields = ("_F",)

    def __init__(self, F, p=None, device="cuda", dtype=torch.float32):
        shape = tuple(F.shape) if isinstance(F, torch.Tensor) else np.shape(F)
        if len(shape) != 2 or shape[0] != shape[1]:
            raise ValueError(f"DimensionMismatch: LULinear needs a square F, got {shape}")
        F = F.detach() if isinstance(F, torch.Tensor) else torch.as_tensor(np.asarray(F, dtype=np.float64))
        self._F = _dev_f32(F.t(), device, dtype)
        self._p, self._dst = None, None
        if p is not None:
            p = [int(v) for v in (p.tolist() if isinstance(p, torch.Tensor) else np.asarray(p).reshape(-1).tolist())]
            if len(p) != shape[0]:
                raise ValueError(f"DimensionMismatch: LULinear has a {shape[0]} x {shape[0]} F and {len(p)} indices")
            self._p = Permute._from_indices(p) + 1
            self._dst = _dev_i32(self._p - 1, device)

    @classmethod
    def from_matrix(cls, A, device="cuda", dtype=torch.float32):
        """The layer of A's LU factorisation with partial pivoting, computed on the host in float64 (scipy.linalg.lu):
        `LULinear.from_matrix(A)` maps y = A x up to the rounding of F to `dtype` -- Glow's initialisation from a random
        rotation."""
        from scipy.linalg import lu

        A = np.asarray(A.detach().cpu().numpy() if isinstance(A, torch.Tensor) else A, dtype=np.float64)
        if A.ndim != 2 or A.shape[0] != A.shape[1]:
            raise ValueError(f"DimensionMismatch: LULinear.from_matrix needs a square matrix, got {A.shape}")
        P, L, U = lu(A)  # A = P·L·U, so row r of L·U is row argmax(P[:, r]) of A
        return cls(np.tril(L, -1) + U, np.argmax(P, axis=0) + 1, device=device, dtype=dtype)

    @property
    def factors(self) -> torch.Tensor:
        return self._F.t()

    @property
    def L(self) -> UnitLowerTriangular:
        return UnitLowerTriangular(self._F.t())

    @property
    def U(self) -> UpperTriangular:
        return UpperTriangular(self._F.t())

    @property
    def p(self) -> np.ndarray:
        return np.arange(1, self._F.shape[0] + 1) if self._p is None else self._p.copy()

    def to(self, device):
        new = _ParamLayer.to(self, device)
        if self._dst is not None:
            new._dst = self._dst.to(device)
        return new

    def _keepalive(self):
        return (self._F,) if self._dst is None else (self._F, self._dst)

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != self._F.shape[0]:
            raise ValueError(f"DimensionMismatch: LULinear has a {self._F.shape[0]} x {self._F.shape[0]} F, input has {D} dims")
        _check_dtype(self._F, dtype, "LULinear")
        if self._dst is None:
            return [_desc(_lib.SCALE_LU, inverse, p0=self._F)]
        return [_desc(_lib.SCALE_LU, inverse, p0=self._F, i0=self._dst)]

    def __eq__(self, o):
        return isinstance(o, LULinear) and torch.equal(self._F.cpu(), o._F.cpu()) and np.array_equal(self.p, o.p)

    __hash__ = object.__hash__


class MaskedAutoregressive(_ParamLayer):
    """MaskedAutoregressive(W1, c1, W2, c2, degrees=None, activation="tanh", slope=0.0): the affine autoregressive layer of
    MAF (Papamakarios et al. 2017) and IAF (Kingma et al. 2016) with a one-hidden-layer MADE conditioner
    (B2B_AUTOREGRESSIVE_MLP; Float32, D <= 128, H <= 256).  Per column, with 1-based rows r and hidden units k of
    degree m_k, masks M₁[k, r] = (r <= m_k) and M₂[i, k] = M₂[D+i, k] = (m_k < i):

        [s; t] = (M₂⊙W₂)·σ.((M₁⊙W₁)·x + c₁) + c₂,   y = x ⊙ exp.(s) + t,   logjac = Σ s

    so sᵢ, tᵢ depend on x₁..x_{i−1} only.  W1 is (H × D) and W2 (2D × H), rows 1..D of W2 giving s and the rest t; c1
    (H) and c2 (2D) may be None.  σ is tanh or LeakyReLU(slope) as for :class:`MLPConditioner`.  `degrees` are any H
    integers, by default MADE's cyclic m_k = ((k−1) mod max(D−1, 1)) + 1; entries outside the masks are never read.

    The layer itself (IAF: sampling runs it) is one network evaluation; `inverse(layer)` recovers x row by row (MAF is
    a flow of inverse layers: its logpdf runs the forward network, rand the sequential recovery).  Rows are taken in
    natural order: put a :class:`Permute` between layers for another.  The cotangents are keyed W1, c1, W2 and c2.
    `_W1` / `_W2` hold W1 and W2 column-major (their transposes row-major), as the descriptor reads them."""

    def __init__(self, W1, c1, W2, c2, degrees=None, activation="tanh", slope=0.0, device="cuda", dtype=torch.float32):
        if dtype != torch.float32:
            raise TypeError("MaskedAutoregressive: the autoregressive layer runs in Float32 only")
        if activation not in _ACT:
            raise ValueError(f"MaskedAutoregressive: activation must be one of {sorted(_ACT)}, got {activation!r}")
        W1n, W2n = _host32(W1), _host32(W2)
        if W1n.ndim != 2 or W1n.shape[0] == 0 or W1n.shape[1] == 0:
            raise ValueError(f"DimensionMismatch: MaskedAutoregressive W1 must be (H, D), got {W1n.shape}")
        H, D = W1n.shape
        if W2n.shape != (2 * D, H):
            raise ValueError(f"DimensionMismatch: MaskedAutoregressive W2 must be (2D, H) = {(2 * D, H)}, got {W2n.shape}")
        if degrees is None:
            degrees = np.arange(H) % max(D - 1, 1) + 1
        deg = np.asarray(degrees.detach().cpu() if isinstance(degrees, torch.Tensor) else degrees).reshape(-1)
        if deg.shape != (H,):
            raise ValueError(f"DimensionMismatch: MaskedAutoregressive has {H} hidden units and {deg.size} degrees")
        if not np.array_equal(deg, np.round(deg)):
            raise ValueError("MaskedAutoregressive: degrees must be integers")
        self.D, self.H, self.activation, self.slope = D, H, activation, float(slope)
        self._W1 = _dev_f32(np.ascontiguousarray(W1n.T), device)  # column-major (H × D)
        self._W2 = _dev_f32(np.ascontiguousarray(W2n.T), device)  # column-major (2D × H)
        self.c1 = _bias(c1, "c1", H, device)
        self.c2 = _bias(c2, "c2", 2 * D, device)
        self._deg = _dev_i32(deg.astype(np.int64), device)

    @property
    def W1(self) -> torch.Tensor:
        return self._W1.t()

    @property
    def W2(self) -> torch.Tensor:
        return self._W2.t()

    @property
    def degrees(self) -> np.ndarray:
        return self._deg.cpu().numpy().astype(np.int64)

    @property
    def masks(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(M₁ (H × D), M₂ (2D × H)) as boolean tensors on the layer's device."""
        m = self._deg.to(torch.int64)
        r = torch.arange(1, self.D + 1, device=m.device)
        M1 = r[None, :] <= m[:, None]
        M2 = (m[None, :] < r[:, None]).repeat(2, 1)
        return M1, M2

    @property
    def device(self):
        return self._W1.device

    def to(self, device):
        new = object.__new__(MaskedAutoregressive)
        new.__dict__.update(self.__dict__)
        for k in ("_W1", "_W2", "c1", "c2", "_deg"):
            t = getattr(self, k)
            setattr(new, k, None if t is None else t.to(device))
        new._cache = {}
        return new

    def params(self) -> Dict[str, torch.Tensor]:
        return {"W1": self.W1, "c1": self.c1, "W2": self.W2, "c2": self.c2}

    def _tensors(self):
        return tuple(t for t in (self._W1, self.c1, self._W2, self.c2) if t is not None)

    def _keepalive(self):
        return self._tensors() + (self._deg,)

    def _descs(self, inverse, D, dtype=torch.float32):
        if D != self.D:
            raise ValueError(f"DimensionMismatch: MaskedAutoregressive has {self.D} dims, input has {D}")
        _check_dtype(self._W1, dtype, "MaskedAutoregressive")
        return [_desc(_lib.AUTOREGRESSIVE_MLP, inverse, p0=self._W1, p1=self.c1 if self.c1 is not None else 0,
                      p2=self._W2, p3=self.c2 if self.c2 is not None else 0, i0=self._deg, n2=self.H,
                      n3=_ACT[self.activation], f0=self.slope)]

    def __eq__(self, o):
        def same(a, b):
            return (a is None and b is None) or (a is not None and b is not None and torch.equal(a.cpu(), b.cpu()))

        return (isinstance(o, MaskedAutoregressive) and self.activation == o.activation and self.slope == o.slope and
                all(same(getattr(self, k), getattr(o, k)) for k in ("_W1", "_W2", "c1", "c2", "_deg")))

    __hash__ = object.__hash__


class LeakyReLU(_ElementwiseLaw):
    """LeakyReLU(α): x ↦ x if x ≥ 0 else αx, α > 0 (leaky_relu.jl:9-29); inverse = LeakyReLU(1/α) (:16) for a scalar α,
    Inverse(layer) for a trainable vector α[D] (:25-29).  α > 0 is checked here; values reached by training are not
    checked on the device.  Batched logjac is per column (the reference sums over the whole array)."""

    code = _lib.EW_LEAKY_RELU
    α = property(lambda s: s.a)

    def __init__(self, α, device="cuda", dtype=torch.float32):
        self._init_law(α, device, dtype)
        if not (bool((self._a > 0).all()) if self.vector else self._s > 0):
            raise ValueError("LeakyReLU needs α > 0")

    def _scalar_inverse(self):
        return LeakyReLU(1.0 / self.a)


class Logit(Bijector):
    """Logit(a, b): y = logit((x − a)/(b − a)) element-wise, logjac = −Σ log((x − a)(b − x)/(b − a))
    (logit.jl:4-29); scalar bounds; the reference's `bounded flow` building block (docs/src/flows.md:25-36)."""

    def __init__(self, a, b):
        self.a, self.b = float(a), float(b)
        if not self.b > self.a:
            raise ValueError("Logit needs a < b")

    code = _lib.EW_LOGIT

    def _descs(self, inverse, D, dtype=torch.float32):
        return _as_stacked(self, D, dtype)._descs(inverse, D, dtype)

    def __eq__(self, o):
        return isinstance(o, Logit) and (o.a, o.b) == (self.a, self.b)  # logit.jl:12

    __hash__ = object.__hash__


class TruncatedBijector(Bijector):
    """TruncatedBijector(lb, ub) (truncated.jl:4-91): clamp to [lb, ub], then logit((x−lb)/(ub−lb)) / log(x−lb) /
    log(ub−x) / identity depending on which bounds are finite (±inf allowed); scalar bounds."""

    def __init__(self, lb, ub):
        self.a, self.b = float(lb), float(ub)
        if not self.b > self.a:
            raise ValueError("TruncatedBijector needs lb < ub")

    lb = property(lambda s: s.a)
    ub = property(lambda s: s.b)
    code = _lib.EW_TRUNCATED

    def _descs(self, inverse, D, dtype=torch.float32):
        return _as_stacked(self, D, dtype)._descs(inverse, D, dtype)

    def __eq__(self, o):
        return isinstance(o, TruncatedBijector) and (o.a, o.b) == (self.a, self.b)

    __hash__ = object.__hash__


class Stacked(Transform):
    """Stacked(bs, ranges): bs[i] applied to rows ranges[i] (1-based inclusive (lo, hi) like Julia
    UnitRanges; stacked.jl:25-59).  Device scope: elementwise blocks (exp, log, identity, Shift, Scale, LeakyReLU,
    Logit, TruncatedBijector)."""

    def __init__(self, bs, ranges=None, device="cuda", dtype=torch.float32):
        bs = list(bs)
        if ranges is None:
            ranges = [(i + 1, i + 1) for i in range(len(bs))]  # Stacked(bs...) = ranges i:i (:49)
        ranges = [(int(lo), int(hi)) for lo, hi in ranges]
        if len(bs) != len(ranges):
            raise ValueError("length(bs) == length(ranges) needs to be true")
        for b in bs:
            if not isinstance(b, (Elementwise, Shift, Scale, LeakyReLU, Logit, TruncatedBijector)) and b is not None:
                raise B2BError(_lib.B2B_EUNSUPPORTED, f"Stacked block {type(b).__name__}")
            if isinstance(b, Scale) and b._A is not None:
                raise B2BError(_lib.B2B_EUNSUPPORTED, "Stacked block Scale with a matrix (a dense layer acts on whole columns)")
            if isinstance(b, _ElementwiseLaw) and b.vector:
                raise B2BError(_lib.B2B_EUNSUPPORTED, f"Stacked block {type(b).__name__} with a vector (one law on whole columns)")
        self.bs, self.ranges_in = bs, ranges
        self.length_in = sum(hi - lo + 1 for lo, hi in ranges)
        self.length_out = self.length_in
        code = np.zeros(self.length_in, np.int32)
        a = np.zeros(self.length_in, np.float64)
        b2 = np.zeros(self.length_in, np.float64)
        for b, (lo, hi) in zip(bs, ranges):
            code[lo - 1:hi] = _lib.EW_IDENTITY if b is None else b.code
            a[lo - 1:hi] = 0.0 if b is None else b.a
            b2[lo - 1:hi] = getattr(b, "b", 0.0) if b is not None else 0.0
        self._code = _dev_i32(code, device)
        self._a = _dev_f32(a.astype(np.float64), device, dtype) if dtype == torch.float64 else _dev_f32(a, device)
        self._b = _dev_f32(b2.astype(np.float64), device, dtype) if dtype == torch.float64 else _dev_f32(b2, device)
        self._dtype = dtype

    def _keepalive(self):
        return (self._code, self._a, self._b)

    def to(self, device):
        new = object.__new__(Stacked)
        new.__dict__.update(self.__dict__)
        new._code, new._a, new._b = self._code.to(device), self._a.to(device), self._b.to(device)
        return new

    @property
    def device(self):
        return self._code.device

    def _descs(self, inverse, D, dtype=torch.float32):
        if self.length_in != D:
            raise RuntimeError(f"input length mismatch ({self.length_in} != {D})")  # stacked.jl:158-160,243-245
        _check_dtype(self._a, dtype, "Stacked")
        return [_desc(_lib.STACKED_EW, inverse, i0=self._code, p0=self._a, p1=self._b)]
