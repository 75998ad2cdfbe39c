"""torch.autograd glue: makes ``with_logabsdet_jacobian`` of a PlanarLayer chain (either direction), of the other per-kind
modules and -- through ``Flow`` -- of any chain differentiable by routing the backward pass to the library's VJP entry
points (``b2b_planar_chain_vjp_f32`` ... ``b2b_chain_vjp_f32``) -- the role the AD extensions play for the
reference (ext/BijectorsChainRulesCoreExt.jl, docs/src/flows.md:93-100).  No arithmetic on batches happens here."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import B2BError
from .interface import (Composed, Inverse, _chain_vjp_raw, _trainable_slots, batchnorm_train_vjp, batchnorm_vjp, colmajor_empty,
                        coupling_vjp, flatten, inverse, planar_chain_vjp, radial_chain_vjp, rqs_vjp, run_chain)
from .layers import (AffineConditioner, Coupling, InvertibleBatchNorm, LULinear, MaskedAutoregressive, PartitionMask, PlanarLayer, RadialLayer,
                     RationalQuadraticSpline, Scale, _ElementwiseLaw)


_VJP_DIMS = (32, 64, 128)


def _colmajor(t: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """A (D, N) tensor with strides (1, D) (no copy when it already has them; a copy is made in ``dtype``)."""
    if t.dim() == 2 and t.stride(0) == 1 and (t.shape[1] == 1 or t.stride(1) == t.shape[0]):
        return t
    out = colmajor_empty(t.shape[0], t.shape[1], t.device, dtype=dtype)
    out.copy_(t)
    return out


class _PlanarChainFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, inv: bool, *wub):
        L = len(wub) // 3
        layers = [PlanarLayer(wub[3 * l].detach(), wub[3 * l + 1].detach(), wub[3 * l + 2].detach()) for l in range(L)]
        flow = Composed(*layers)
        t = inverse(flow) if inv else flow
        xc = _colmajor(x.detach())
        y, lj = run_chain(t, xc)
        ctx.t, ctx.inv, ctx.L, ctx.layers = t, inv, L, layers
        ctx.save_for_backward(xc)
        return y, lj

    @staticmethod
    def backward(ctx, ybar, ljbar):
        (xc,) = ctx.saved_tensors
        D, N = xc.shape
        yb = _colmajor(ybar) if ybar is not None else _colmajor(torch.zeros((D, N), device=xc.device))
        lb = ljbar.contiguous() if ljbar is not None else None
        t = ctx.t
        Dp = next((d for d in _VJP_DIMS if d >= D), None)
        if Dp is None:
            raise NotImplementedError(f"planar VJP kernels cover D <= {_VJP_DIMS[-1]} (got {D})")
        if Dp != D:
            # The reverse-mode kernels are built for D in {32, 64, 128}.  A planar layer on zero-padded rows is the same
            # map (w, u padded with zeros: wᵀz, wᵀu, ‖w‖² and the first D rows of û are unchanged), so smaller flows
            # (the reference's own example is D = 2, docs/src/flows.md:40-60) run embedded in the next supported D.
            pad = lambda v: torch.cat([v, v.new_zeros(Dp - D)])
            layers = [PlanarLayer(pad(l.w), pad(l.u), l.b) for l in ctx.layers]
            t = inverse(Composed(*layers)) if ctx.inv else Composed(*layers)
            xp, ybp = colmajor_empty(Dp, N, xc.device), colmajor_empty(Dp, N, xc.device)
            xp.zero_()
            ybp.zero_()
            xp[:D].copy_(xc)
            ybp[:D].copy_(yb)
            xc, yb = xp, ybp
        xbar, grads = planar_chain_vjp(t, xc, yb, lb)
        if Dp != D:
            xbar = xbar[:D]
            grads = [{"w": g["w"][:D], "u": g["u"][:D], "b": g["b"]} for g in grads]
        if ctx.inv:  # application order of inverse(flow) is the flow's layers reversed
            grads = grads[::-1]
        flat: List[torch.Tensor] = []
        for g in grads:
            flat += [g["w"], g["u"], g["b"]]
        return (xbar, None, *flat)


class PlanarFlow(torch.nn.Module):
    """A trainable ∘-chain of L PlanarLayers (planar_layer.jl:13-28: randn-initialised w, u, b) on the device."""

    def __init__(self, dims: int, n_layers: int, device="cuda", generator=None, scale: float = 1.0):
        super().__init__()
        mk = lambda n: torch.nn.Parameter((torch.randn(n, generator=generator) * scale).to(device))
        self.w = torch.nn.ParameterList([mk(dims) for _ in range(n_layers)])
        self.u = torch.nn.ParameterList([mk(dims) for _ in range(n_layers)])
        self.b = torch.nn.ParameterList([mk(1) for _ in range(n_layers)])

    def _wub(self) -> Sequence[torch.Tensor]:
        out = []
        for w, u, b in zip(self.w, self.u, self.b):
            out += [w, u, b]
        return out

    def layers(self) -> List[PlanarLayer]:
        return [PlanarLayer(w.detach(), u.detach(), b.detach()) for w, u, b in zip(self.w, self.u, self.b)]

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """with_logabsdet_jacobian(flow, x), differentiable w.r.t. x and the parameters."""
        return _PlanarChainFn.apply(x, False, *self._wub())

    def inverse(self, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """with_logabsdet_jacobian(inverse(flow), y), differentiable (find_alpha through its implicit rule)."""
        return _PlanarChainFn.apply(y, True, *self._wub())


class _RadialChainFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, inv: bool, *abz):
        L = len(abz) // 3
        flow = Composed(*[RadialLayer(abz[3 * l].detach(), abz[3 * l + 1].detach(), abz[3 * l + 2].detach()) for l in range(L)])
        t = inverse(flow) if inv else flow
        xc = _colmajor(x.detach())
        y, lj = run_chain(t, xc)
        ctx.t, ctx.inv = t, inv
        ctx.save_for_backward(xc)
        return y, lj

    @staticmethod
    def backward(ctx, ybar, ljbar):
        (xc,) = ctx.saved_tensors
        D, N = xc.shape
        yb = _colmajor(ybar) if ybar is not None else _colmajor(torch.zeros((D, N), device=xc.device))
        xbar, grads = radial_chain_vjp(ctx.t, xc, yb, ljbar.contiguous() if ljbar is not None else None)
        if ctx.inv:  # application order of inverse(flow) is the flow's layers reversed
            grads = grads[::-1]
        flat: List[torch.Tensor] = []
        for g in grads:
            flat += [g["α_"], g["β"], g["z_0"]]
        return (xbar, None, *flat)


class RadialFlow(torch.nn.Module):
    """A trainable ∘-chain of L RadialLayers (radial_layer.jl:11-27: randn-initialised α_, β, z_0), forward direction
    (the sampling / variational path): ``with_logabsdet_jacobian`` differentiable w.r.t. x and the raw parameters."""

    def __init__(self, dims: int, n_layers: int, device="cuda", generator=None):
        super().__init__()
        mk = lambda n: torch.nn.Parameter(torch.randn(n, generator=generator).to(device))
        self.alpha_ = torch.nn.ParameterList([mk(1) for _ in range(n_layers)])
        self.beta = torch.nn.ParameterList([mk(1) for _ in range(n_layers)])
        self.z_0 = torch.nn.ParameterList([mk(dims) for _ in range(n_layers)])

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        return _RadialChainFn.apply(x, False, *self._abz())

    def _abz(self):
        abz = []
        for a, b, z in zip(self.alpha_, self.beta, self.z_0):
            abz += [a, b, z]
        return abz

    def inverse(self, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """with_logabsdet_jacobian(inverse(flow), y), differentiable (compute_r through its implicit rule): the
        logpdf / NLL path of a radial flow."""
        return _RadialChainFn.apply(y, True, *self._abz())


# ---- RealNVP: affine Coupling + eval-mode InvertibleBatchNorm blocks (BASELINE config 5) ---------------------------------
class _CouplingFn(torch.autograd.Function):
    """with_logabsdet_jacobian of ONE affine coupling layer (either direction); backward = b2b_coupling_affine_vjp_f32."""

    @staticmethod
    def forward(ctx, x, W, c, mask, inv: bool):
        cond = AffineConditioner.__new__(AffineConditioner)
        cond.n1, cond.n2 = W.shape[0] // 2, W.shape[1]
        cond.W, cond.c = W.detach().t().contiguous(), c.detach().contiguous()  # device layout: column-major (2n1 × n2)
        lay = Coupling(cond, mask)
        t = inverse(lay) if inv else lay
        xc = _colmajor(x.detach())
        y, lj = run_chain(t, xc)
        ctx.t = t
        ctx.save_for_backward(xc)
        return y, lj

    @staticmethod
    def backward(ctx, ybar, ljbar):
        (xc,) = ctx.saved_tensors
        D, N = xc.shape
        yb = _colmajor(ybar) if ybar is not None else _colmajor(torch.zeros((D, N), device=xc.device))
        xbar, g = coupling_vjp(ctx.t, xc, yb, ljbar.contiguous() if ljbar is not None else None)
        return xbar, g["W"], g["c"], None, None


class _BatchNormFn(torch.autograd.Function):
    """with_logabsdet_jacobian of ONE eval-mode InvertibleBatchNorm (either direction); backward = b2b_batchnorm_eval_vjp_f32."""

    @staticmethod
    def forward(ctx, x, b, logs, m, v, eps: float, inv: bool):
        lay = InvertibleBatchNorm(b=b.detach(), logs=logs.detach(), m=m, v=v, eps=eps, device=x.device)
        t = inverse(lay) if inv else lay
        xc = _colmajor(x.detach())
        y, lj = run_chain(t, xc)
        ctx.t = t
        ctx.save_for_backward(xc)
        return y, lj

    @staticmethod
    def backward(ctx, ybar, ljbar):
        (xc,) = ctx.saved_tensors
        D, N = xc.shape
        yb = _colmajor(ybar) if ybar is not None else _colmajor(torch.zeros((D, N), device=xc.device))
        xbar, g = batchnorm_vjp(ctx.t, xc, yb, ljbar.contiguous() if ljbar is not None else None)
        return xbar, g["b"], g["logs"], None, None, None, None


class _BatchNormTrainFn(torch.autograd.Function):
    """with_logabsdet_jacobian of ONE training-mode InvertibleBatchNorm (normalise.jl:51-67): the forward runs
    b2b_batchnorm_train_fwd_f32 once (so the moving statistics move once per step); backward = b2b_batchnorm_train_vjp_f32,
    which recomputes the batch statistics from the saved x and leaves the moving statistics alone."""

    @staticmethod
    def forward(ctx, x, b, logs, m, v, eps: float, mtm: float, comm):
        lay = InvertibleBatchNorm(b=b.detach(), logs=logs.detach(), m=m, v=v, eps=eps, mtm=mtm, device=x.device, training=True)
        xc = _colmajor(x.detach())
        y, lj = lay.train_forward(xc, comm)
        ctx.lay, ctx.comm = lay, comm
        ctx.save_for_backward(xc)
        return y, lj

    @staticmethod
    def backward(ctx, ybar, ljbar):
        (xc,) = ctx.saved_tensors
        yb = _colmajor(ybar) if ybar is not None else None
        xbar, g = batchnorm_train_vjp(ctx.lay, xc, yb, ljbar.contiguous() if ljbar is not None else None, ctx.comm)
        return xbar, g["b"], g["logs"], None, None, None, None, None


class TrainingBatchNorm(torch.nn.Module):
    """A trainable InvertibleBatchNorm(dims; eps, mtm) in training mode (normalise.jl:26-37,51-67): parameters ``b``,
    ``logs``; buffers ``m``, ``v`` (the moving statistics, updated once per forward).  ``forward(x)`` returns (y, logjac)
    computed with the batch statistics -- over all ranks of ``comm`` (a distributed.Communicator) when given --
    differentiable w.r.t. x, b and logs.  With ``comm``, the b / logs gradients are this rank's share: all-reduce them with
    the rest of the gradient.  The layer has no inverse in training mode (normalise.jl:75)."""

    def __init__(self, dims: int, comm=None, eps: float = 1e-5, mtm: float = 1e-1, device="cuda"):
        super().__init__()
        self.comm, self.eps, self.mtm = comm, float(np.float32(eps)), float(np.float32(mtm))
        self.b = torch.nn.Parameter(torch.zeros(dims, device=device))
        self.logs = torch.nn.Parameter(torch.zeros(dims, device=device))
        self.register_buffer("m", torch.zeros(dims, device=device))
        self.register_buffer("v", torch.ones(dims, device=device))

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        return _BatchNormTrainFn.apply(x, self.b, self.logs, self.m, self.v, self.eps, self.mtm, self.comm)


_NO_TRAINING_INVERSE = "`with_logabsdet_jacobian(::Inverse{InvertibleBatchNorm})` is only available in test mode."  # normalise.jl:75


class RealNVP(torch.nn.Module):
    """A trainable RealNVP flow: `n_blocks` x (affine Coupling with alternating half masks + eval-mode InvertibleBatchNorm),
    the structure of BASELINE config 5.  ``forward(x)`` / ``inverse(y)`` return (result, logjac), differentiable w.r.t.
    the input and the parameters W, c (conditioners) and b, logs (BatchNorm; m, v are statistics); ``nll(y)`` is the
    training objective of docs/src/flows.md:74-77 with a standard-normal base.
    ``batchnorm_training=True`` puts the BatchNorm layers in training mode (istraining() == true, normalise.jl:51-67):
    ``forward`` then normalises with the batch statistics, updates ``m`` / ``v`` once per call and differentiates through
    the statistics; ``inverse`` and ``nll`` raise, as the reference asserts at normalise.jl:75."""

    def __init__(self, dims: int, n_blocks: int, device="cuda", generator=None, scale: float = 0.05,
                 batchnorm_training: bool = False):
        super().__init__()
        self.batchnorm_training = batchnorm_training
        h = dims // 2
        self.dims, self.masks = dims, []
        Ws, cs, bs, ls = [], [], [], []
        for l in range(n_blocks):
            first = l % 2 == 0
            idx1 = list(range(1, h + 1)) if first else list(range(h + 1, dims + 1))
            idx2 = list(range(h + 1, dims + 1)) if first else list(range(1, h + 1))
            self.masks.append(PartitionMask(dims, idx1, idx2))
            n1, n2 = len(idx1), len(idx2)
            Ws.append(torch.nn.Parameter((torch.randn((2 * n1, n2), generator=generator) * scale / n2 ** 0.5).to(device)))
            cs.append(torch.nn.Parameter(torch.zeros(2 * n1, device=device)))
            bs.append(torch.nn.Parameter(torch.zeros(dims, device=device)))
            ls.append(torch.nn.Parameter(torch.zeros(dims, device=device)))
        self.W, self.c = torch.nn.ParameterList(Ws), torch.nn.ParameterList(cs)
        self.b, self.logs = torch.nn.ParameterList(bs), torch.nn.ParameterList(ls)
        self.register_buffer("m", torch.zeros(n_blocks, dims, device=device))
        self.register_buffer("v", torch.ones(n_blocks, dims, device=device))
        self.eps, self.mtm = 1e-5, float(np.float32(1e-1))

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        lj = None
        for l in range(len(self.W)):
            x, l1 = _CouplingFn.apply(x, self.W[l], self.c[l], self.masks[l], False)
            if self.batchnorm_training:
                x, l2 = _BatchNormTrainFn.apply(x, self.b[l], self.logs[l], self.m[l], self.v[l], self.eps, self.mtm, None)
            else:
                x, l2 = _BatchNormFn.apply(x, self.b[l], self.logs[l], self.m[l], self.v[l], self.eps, False)
            lj = l1 + l2 if lj is None else lj + l1 + l2
        return x, lj

    def inverse(self, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        if self.batchnorm_training:
            raise AssertionError(_NO_TRAINING_INVERSE)
        lj = None
        for l in reversed(range(len(self.W))):
            y, l2 = _BatchNormFn.apply(y, self.b[l], self.logs[l], self.m[l], self.v[l], self.eps, True)
            y, l1 = _CouplingFn.apply(y, self.W[l], self.c[l], self.masks[l], True)
            lj = l1 + l2 if lj is None else lj + l1 + l2
        return y, lj

    def nll(self, y: torch.Tensor) -> torch.Tensor:
        """−Σ_n logpdf(transformed(MvNormal(0, I), flow), y_n) (transformed_distribution.jl:165-169)."""
        x, lj = self.inverse(y)
        base = -0.5 * (x * x).sum(0) - 0.5 * self.dims * 1.8378770664093453
        return -(base + lj).sum()


# ---- RationalQuadraticSpline -------------------------------------------------------------------------------------------
class _SplineFn(torch.autograd.Function):
    """with_logabsdet_jacobian of ONE RationalQuadraticSpline given its PROCESSED knots (D × K+1 each), either direction;
    backward = b2b_rqs_vjp_f32 (cotangents of the input and of the three knot arrays)."""

    @staticmethod
    def forward(ctx, x, widths, heights, derivs, inv: bool):
        lay = RationalQuadraticSpline(widths.detach(), heights.detach(), derivs.detach(), device=x.device)
        t = inverse(lay) if inv else lay
        xc = _colmajor(x.detach())
        y, lj = run_chain(t, xc)
        ctx.t = t
        ctx.save_for_backward(xc)
        return y, lj

    @staticmethod
    def backward(ctx, ybar, ljbar):
        (xc,) = ctx.saved_tensors
        D, N = xc.shape
        yb = _colmajor(ybar) if ybar is not None else _colmajor(torch.zeros((D, N), device=xc.device))
        xbar, g = rqs_vjp(ctx.t, xc, yb, ljbar.contiguous() if ljbar is not None else None)
        return xbar, g["widths"], g["heights"], g["derivatives"], None


class SplineLayer(torch.nn.Module):
    """A trainable RationalQuadraticSpline(raw widths, raw heights, raw derivatives, B) (rational_quadratic_spline.jl:
    99-123).  The constructor's normalisation (softmax -> cumsum -> [-B, B] knots, softplus derivatives with unit end
    slopes) is parameter-sized torch code, differentiated by torch as the reference's AD differentiates the constructor;
    the spline over the batch and its reverse mode run in the device kernels."""

    def __init__(self, dims: int, K: int, B: float = 3.0, device="cuda", generator=None):
        super().__init__()
        self.B = float(B)
        self.w = torch.nn.Parameter(torch.randn((dims, K), generator=generator).to(device))
        self.h = torch.nn.Parameter(torch.randn((dims, K), generator=generator).to(device))
        self.d = torch.nn.Parameter(torch.randn((dims, K - 1), generator=generator).to(device))

    def knots(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        n, dev = self.w.shape[0], self.w.device
        zero, one = torch.zeros((n, 1), device=dev), torch.ones((n, 1), device=dev)
        W = 2 * self.B * torch.cumsum(torch.cat([zero, torch.softmax(self.w, dim=1)], dim=1), dim=1) - self.B
        H = 2 * self.B * torch.cumsum(torch.cat([zero, torch.softmax(self.h, dim=1)], dim=1), dim=1) - self.B
        Dv = torch.cat([one, torch.nn.functional.softplus(self.d), one], dim=1)
        return W, H, Dv

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        return _SplineFn.apply(x, *self.knots(), False)

    def inverse(self, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        return _SplineFn.apply(y, *self.knots(), True)


# ---- any chain: one b2b_chain_vjp_f32 (Float64: b2b_chain_vjp_f64) call per backward -------------------------------------
def _trainable_tensors(leaf) -> List[torch.Tensor]:
    """The device tensors of a leaf's trainable fields (Functors' trainable set of the reference's layer structs)."""
    lay = leaf.orig if isinstance(leaf, Inverse) else leaf
    if isinstance(lay, PlanarLayer):
        return [lay.w, lay.u, lay.b]
    if isinstance(lay, RadialLayer):
        return [getattr(lay, "α_"), getattr(lay, "β"), lay.z_0]
    if isinstance(lay, RationalQuadraticSpline):
        return [lay.widths, lay.heights, lay.derivatives]
    if isinstance(lay, Coupling):
        return [t for t in lay.θ._tensors() if t is not None]
    if isinstance(lay, Scale) and lay._A is not None:  # dense or triangular matrix
        return [lay._A]
    if isinstance(lay, LULinear):
        return [lay._F]
    if isinstance(lay, MaskedAutoregressive):
        return list(lay._tensors())
    if isinstance(lay, _ElementwiseLaw) and lay.vector:  # Shift / Scale / LeakyReLU with a vector parameter
        return [lay._a]
    if isinstance(lay, InvertibleBatchNorm):
        if lay.training:
            raise B2BError(_lib.B2B_EUNSUPPORTED, "Flow: InvertibleBatchNorm in training mode has no reverse mode on the device")
        return [lay.b, lay.logs]
    return []


class _ChainFn(torch.autograd.Function):
    """with_logabsdet_jacobian of a whole chain (plus, for logpdf, the terminal MvNormal); backward = ONE
    b2b_chain_vjp_f32 call (b2b_chain_vjp_f64 for Float64 batches) whose parameter cotangents are routed to the parameters
    by device address."""

    @staticmethod
    def forward(ctx, x, t, extra, want_y: bool, *params):
        xc = _colmajor(x.detach(), x.dtype)
        D = xc.shape[0]
        y, lj = run_chain(t, xc, want_y=want_y, extra_descs=extra)
        descs = list(t._descs(False, D, xc.dtype)) + list(extra)
        owner = {p.data_ptr(): k for k, p in enumerate(params) if ctx.needs_input_grad[4 + k]}
        # a parameter can appear in several descriptors (a layer used twice): its cotangent is the sum
        ctx.want = [(l, i, owner[getattr(d, f"p{i}")]) for l, d in enumerate(descs) for i in _trainable_slots(d)
                    if getattr(d, f"p{i}") in owner]
        ctx.t, ctx.descs, ctx.extra, ctx.want_y, ctx.shapes = t, descs, extra, want_y, [p.shape for p in params]
        ctx.save_for_backward(xc)
        return (y, lj) if want_y else lj

    @staticmethod
    def backward(ctx, *grads):
        (xc,) = ctx.saved_tensors
        ybar, ljbar = grads if ctx.want_y else (None, grads[0])
        yb = _colmajor(ybar, xc.dtype) if ybar is not None else None
        lb = ljbar.contiguous() if ljbar is not None else None
        xbar, bars = _chain_vjp_raw(ctx.descs, xc, yb, lb, [(l, i) for l, i, _ in ctx.want])
        out: List = [None] * len(ctx.shapes)
        for l, i, k in ctx.want:
            g = bars[(l, i)].reshape(ctx.shapes[k])
            out[k] = g if out[k] is None else out[k] + g
        return (xbar, None, None, None, *out)


class _RSampleFn(torch.autograd.Function):
    """rand_logpdf of a transformed base, differentiable in the flow's and the base's parameters with the draw z held
    fixed; backward = ONE b2b_chain_sample_vjp_f32 call whose cotangents are routed to the parameters by device address.
    The seed of the forward is kept for the backward."""

    @staticmethod
    def forward(ctx, td, n: int, seed: int, offset: int, column_offset: int, *params):
        from .transformed_distribution import _rsample_setup, rand_logpdf

        y, lq = rand_logpdf(td, n, seed, offset, column_offset)
        dist, descs, _, base, dev = _rsample_setup(td, n, "rsample")
        full = list(descs) + [base]
        owner = {p.data_ptr(): k for k, p in enumerate(params) if ctx.needs_input_grad[5 + k]}
        ctx.want = [(l, i, owner[getattr(d, f"p{i}")]) for l, d in enumerate(full) for i in _trainable_slots(d)
                    if getattr(d, f"p{i}") in owner]
        ctx.descs, ctx.base, ctx.D, ctx.n, ctx.dev = descs, base, dist.D, int(n), dev
        ctx.seed, ctx.offset, ctx.column_offset, ctx.shapes = seed, offset, column_offset, [p.shape for p in params]
        return y, lq

    @staticmethod
    def backward(ctx, ybar, lqbar):
        from .transformed_distribution import _rand_vjp_raw

        yb = _colmajor(ybar) if ybar is not None else None
        lb = lqbar.contiguous() if lqbar is not None else None
        bars = _rand_vjp_raw(ctx.descs, ctx.base, ctx.D, ctx.n, ctx.dev, yb, lb, ctx.seed, ctx.offset,
                             ctx.column_offset, [(l, i) for l, i, _ in ctx.want])
        out: List = [None] * len(ctx.shapes)
        for l, i, k in ctx.want:
            g = bars[(l, i)].reshape(ctx.shapes[k])
            out[k] = g if out[k] is None else out[k] + g
        return (None, None, None, None, None, *out)


class Flow(torch.nn.Module):
    """A trainable flow made of ANY chain of the supported layers -- `Stacked(ibs) ∘ PlanarLayer(2)`, spline flows with
    permutations, coupling flows with bounded outputs -- over an optional MvNormal base.  Its parameters are the trainable
    fields of every leaf of ``flatten(transform)`` (w/u/b, α_/β/z_0, processed RQS knots, W/c, b/logs) and μ, σ or μ, L
    (``MvNormal(..., scale_tril=L)``; the parameter holds L column-major, i.e. Lᵀ row-major) of the base when it has them, registered on the leaves' own device storage: an optimiser step is what the next launch reads.
    ``forward(x)`` / ``inverse(y)`` return (result, logjac); ``logpdf(y)`` is logpdf(transformed(base, transform), y) and
    ``nll(y)`` = −Σ logpdf.  Each is one autograd Function whose backward is one b2b_chain_vjp_f32 call.  A flow whose
    layers (and base) are Float64 takes Float64 batches, and its backward is one b2b_chain_vjp_f64 call; a Float32 /
    Float64 mix raises TypeError.  A training-mode InvertibleBatchNorm raises (it has no reverse mode here)."""

    def __init__(self, transform, base=None):
        super().__init__()
        from .transformed_distribution import MvNormal

        self.transform, self.base = transform, base
        tensors, seen = [], set()
        for leaf in flatten(transform):
            for t in _trainable_tensors(leaf):
                if t.data_ptr() not in seen:
                    seen.add(t.data_ptr())
                    tensors.append(t)
        if isinstance(base, MvNormal):
            tensors += [t for t in (base.mu, base.sigma, base._tril) if t is not None]
        self.params = torch.nn.ParameterList([torch.nn.Parameter(t) for t in tensors])  # shares the leaves' storage

    def _base(self, D, device, dtype=torch.float32):
        from .transformed_distribution import MvNormal

        return self.base if self.base is not None else MvNormal(D, device=device, dtype=dtype)

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        return _ChainFn.apply(x, self.transform, (), True, *self.params)

    def inverse(self, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        return _ChainFn.apply(y, inverse(self.transform), (), True, *self.params)

    def logpdf(self, y: torch.Tensor) -> torch.Tensor:
        term = self._base(y.shape[0], y.device, y.dtype)._terminal_desc()
        return _ChainFn.apply(y, inverse(self.transform), (term,), False, *self.params)

    def nll(self, y: torch.Tensor) -> torch.Tensor:
        return -self.logpdf(y).sum()

    def rsample(self, n: int, seed=None, offset: int = 0, column_offset: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """``(y, logq)`` = rand_logpdf(transformed(base, transform), n, ...): n samples of the flow and their log-density,
        differentiable in ``params`` -- the flow's and the base's μ, σ or L -- with the base draw held fixed (the
        reparameterisation gradient of an ELBO, docs/src/advi.md).  The backward is one b2b_chain_sample_vjp_f32 call
        with the forward's seed (``seed=None`` draws one, once).  Float32 only; the flow needs an MvNormal base."""
        from .transformed_distribution import MvNormal, _seed, transformed

        if not isinstance(self.base, MvNormal):
            raise ValueError("Flow.rsample: the flow has no base distribution; construct it with Flow(transform, MvNormal(D, ...))")
        td = transformed(self.base, self.transform)
        return _RSampleFn.apply(td, int(n), _seed(seed), int(offset), int(column_offset), *self.params)
