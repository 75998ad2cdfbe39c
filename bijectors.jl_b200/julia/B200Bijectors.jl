# B200Bijectors.jl -- the reference-side binding of libb2b.so (include/b2b.h).
#
# This is the file a Bijectors.jl maintainer adds as a PACKAGE EXTENSION of Bijectors.jl on CUDA.jl
# (ext/BijectorsB200Ext.jl; `[weakdeps] CUDA`, `[extensions] BijectorsB200Ext = "CUDA"`), so every method below is a
# more specific method of Bijectors' OWN generic functions on Bijectors' OWN layer types parametrised by CuArrays --
# no type piracy.  Bijectors.jl has no FFI/plugin registry: "plugging in" = dispatch (src/interface.jl:144,156,183,265).
# Not exercised by the test suite (it has no Julia toolchain); the identical C ABI is exercised by the
# Python/ctypes harness in bijectors.jl_b200/ (tests/, bench.py), and tests/test_host_logic.py parses every `ccall` in
# this file and checks symbol, arity and argument classes against include/b2b.h.
#
# Conventions (include/b2b.h): D×N Float32 CuMatrix batches (Julia is column-major, so a column is one sample);
# every pointer is a device pointer unless the C name says host; the stream is CUDA.jl's task-local stream; non-zero
# status -> error(b2b_status_string(rc)).
module B200Bijectors

using CUDA
using Bijectors
using Bijectors: PlanarLayer, RadialLayer, RationalQuadraticSpline, Coupling, PartitionMask, InvertibleBatchNorm,
                 Permute, Stacked, Shift, Scale, LeakyReLU, Logit, TruncatedBijector, Inverse, TransformedDistribution
import Bijectors: transform, logabsdetjac, with_logabsdet_jacobian
import Distributions
using Distributions: MvNormal
using PDMats: PDMat, PDiagMat, ScalMat
using LinearAlgebra: LowerTriangular, UpperTriangular, UnitLowerTriangular, UnitUpperTriangular, cholesky, diagind
using Functors: fmap
using SparseArrays: findnz
using Statistics: mean, var
import ChainRulesCore
using ChainRulesCore: NoTangent

const libb2b = get(ENV, "LIBB2B", "libb2b.so")

# ---- b2b_layer_desc (include/b2b.h) ------------------------------------------------------------------
struct LayerDesc
    kind::Int32
    inverse::Int32
    n0::Int32; n1::Int32; n2::Int32; n3::Int32
    f0::Float32; f1::Float32
    p0::CuPtr{Float32}; p1::CuPtr{Float32}; p2::CuPtr{Float32}; p3::CuPtr{Float32}
    i0::CuPtr{Int32}; i1::CuPtr{Int32}
end
const PLANAR, RADIAL, RQS, COUPLING_AFFINE, BATCHNORM, PERMUTE, STACKED_EW, MVNORMAL_DIAG, MVNORMAL_TRIL = Int32.(1:9)
const COUPLING_RQS = Int32(11)  # 10 is not a layer kind (include/b2b.h)
const SCALE_MATRIX = Int32(12)
const COUPLING_MLP = Int32(13)
const COUPLING_MLP_RQS = Int32(14)
const COUPLING_DEEP_MLP = Int32(15)
const COUPLING_DEEP_MLP_RQS = Int32(16)
const ELEMENTWISE_VEC = Int32(17)
const SCALE_TRIANGULAR = Int32(18)
const SCALE_TRIANGULAR_MAX_D = 256
const SCALE_LU = Int32(19)
const SCALE_LU_MAX_D = 256
const AUTOREGRESSIVE_MLP = Int32(20)
const AUTOREGRESSIVE_MLP_MAX_D = 128
const AUTOREGRESSIVE_MLP_MAX_H = 256
const ACT_TANH, ACT_LEAKY_RELU = Int32(0), Int32(1)
const EW_IDENTITY, EW_EXP, EW_LOG, EW_SHIFT, EW_SCALE, EW_LEAKY_RELU, EW_LOGIT, EW_TRUNCATED = Int32.(0:7)
const NULLF = CuPtr{Float32}(0)
const NULLI = CuPtr{Int32}(0)

check(rc::Cint) = rc == 0 ? nothing :
    error(unsafe_string(ccall((:b2b_status_string, libb2b), Cstring, (Cint,), rc)))

stream_handle() = CUDA.stream().handle

# Device placement of a flow is the reference's own mechanism: Functors.fmap(cu, flow)
# (Functors.@functor PlanarLayer / RadialLayer / InvertibleBatchNorm (b, logs) / Inverse; SURVEY §5).
to_device(flow) = fmap(x -> x isa AbstractArray{<:Real} ? cu(Float32.(x)) : x, flow)

# ---- layer -> descriptor ------------------------------------------------------------------------------
# Parameters are passed RAW (the struct fields); û, wᵀû, softplus terms are derived on the device.
# A descriptor only holds pointers: `owners(b)` lists the arrays that must stay rooted while a launch is in flight.
desc(b::PlanarLayer{<:CuVector{Float32}}, inv::Bool) =
    LayerDesc(PLANAR, inv, 0, 0, 0, 0, 0f0, 0f0, pointer(b.w), pointer(b.u), pointer(b.b), NULLF, NULLI, NULLI)
desc(b::RadialLayer{<:CuVector{Float32}}, inv::Bool) =
    LayerDesc(RADIAL, inv, 0, 0, 0, 0, 0f0, 0f0, pointer(b.α_), pointer(b.β), pointer(b.z_0), NULLF, NULLI, NULLI)
desc(b::RationalQuadraticSpline{<:CuMatrix{Float32}}, inv::Bool) =       # fields are D×(K+1), column-major
    LayerDesc(RQS, inv, size(b.widths, 2), 0, 0, 0, 0f0, 0f0,
              pointer(b.widths), pointer(b.heights), pointer(b.derivatives), NULLF, NULLI, NULLI)
function desc(b::InvertibleBatchNorm{<:CuVector{Float32}}, inv::Bool)
    Bijectors.istraining() && error("InvertibleBatchNorm in training mode is a separate call: batchnorm_train!")
    LayerDesc(BATCHNORM, inv, 0, 0, 0, 0, Float32(b.eps), 0f0,
              pointer(b.b), pointer(b.logs), pointer(b.m), pointer(b.v), NULLI, NULLI)
end
desc(b::Inverse, inv::Bool) = desc(b.orig, !inv)

# The recognised coupling law θ(x₂) = Shift(t) ∘ Scale(exp.(s)), [s;t] = W*x₂ .+ c (SURVEY §8 a12).
struct AffineConditioner{M<:CuMatrix{Float32},V<:CuVector{Float32}}
    W::M   # (2n1 × n2)
    c::V
end
(θ::AffineConditioner)(x₂) = (st = θ.W * x₂ .+ θ.c; n = length(st) ÷ 2;
                              Shift(st[(n + 1):end]) ∘ Scale(exp.(st[1:n])))
# Device-side tables (index lists, elementwise codes) are built once per host object and cached, so that they outlive
# every launch that uses them.
struct DeviceMask            # index lists of a PartitionMask (coupling.jl:51-118), 0-based on the device
    idx1::CuVector{Int32}; idx2::CuVector{Int32}; row1::Int32; row2::Int32
end
function DeviceMask(m::PartitionMask)
    rows(A) = Int32.(findnz(A)[1] .- 1)          # A_i[idx, j] = 1
    first_row(r) = (length(r) > 0 && r == collect(r[1]:(r[1] + length(r) - 1))) ? r[1] : Int32(-1)
    r1, r2 = rows(m.A_1), rows(m.A_2)
    DeviceMask(cu(r1), cu(r2), first_row(r1), first_row(r2))
end
const MASKS = IdDict{Any,DeviceMask}()
function desc(cl::Coupling{<:AffineConditioner}, inv::Bool)
    dm = get!(() -> DeviceMask(cl.mask), MASKS, cl.mask)
    LayerDesc(COUPLING_AFFINE, inv, length(dm.idx1), length(dm.idx2), dm.row1, dm.row2, 0f0, 0f0,
              pointer(cl.θ.W), pointer(cl.θ.c), NULLF, NULLF, pointer(dm.idx1), pointer(dm.idx2))
end
# The neural-spline coupling law (Durkan et al. 2019): θ(x₂) = RationalQuadraticSpline(reshape(v[1:n1K], n1, K),
# reshape(v[n1K+1:2n1K], n1, K), reshape(v[2n1K+1:end], n1, K−1), B) with v = W*x₂ .+ c -- the reference's own normalising
# constructor (rational_quadratic_spline.jl:109-123), so the same object also runs on the CPU reference path.  Float32,
# n1, n2 <= 128, 2 <= K <= 16, D <= 1024 on the device; c === nothing is a zero shift.
struct SplineConditioner{M<:AbstractMatrix,V}
    W::M   # ((3K−1)·n1 × n2)
    c::V   # (3K−1)·n1, or nothing
    K::Int
    B::Float32
end
function (θ::SplineConditioner)(x₂)
    v = θ.c === nothing ? θ.W * x₂ : θ.W * x₂ .+ θ.c
    n1, K = size(θ.W, 1) ÷ (3θ.K - 1), θ.K
    RationalQuadraticSpline(reshape(v[1:(n1 * K)], n1, K), reshape(v[(n1 * K + 1):(2n1 * K)], n1, K),
                            reshape(v[(2n1 * K + 1):end], n1, K - 1), θ.B)
end
function desc(cl::Coupling{<:SplineConditioner{<:CuMatrix{Float32}}}, inv::Bool)
    dm = get!(() -> DeviceMask(cl.mask), MASKS, cl.mask)
    θ = cl.θ
    LayerDesc(COUPLING_RQS, inv, length(dm.idx1), length(dm.idx2), θ.K, 0, θ.B, 0f0,
              pointer(θ.W), θ.c === nothing ? NULLF : pointer(θ.c), NULLF, NULLF, pointer(dm.idx1), pointer(dm.idx2))
end
# The neural-network coupling law of RealNVP: θ(x₂) = Shift(t) ∘ Scale(exp.(s)), [s; t] = W₂*σ.(W₁*x₂ .+ c₁) .+ c₂ with
# σ = tanh or LeakyReLU(slope) (x >= 0 ? x : slope*x, leaky_relu.jl:18-29); a callable, so the same object also runs on the
# CPU reference path.  Float32, n1, n2 <= 128, H <= 256, D <= 1024 on the device; c₁ / c₂ === nothing is a zero shift.
struct MLPConditioner{M<:AbstractMatrix,V1,V2}
    W1::M   # (H × n2)
    c1::V1  # H, or nothing
    W2::M   # (2n1 × H)
    c2::V2  # 2n1, or nothing
    act::Int32      # ACT_TANH or ACT_LEAKY_RELU
    slope::Float32
end
function (θ::MLPConditioner)(x₂)
    v = θ.c1 === nothing ? θ.W1 * x₂ : θ.W1 * x₂ .+ θ.c1
    h = θ.act == ACT_TANH ? tanh.(v) : ifelse.(v .>= 0, v, θ.slope .* v)
    st = θ.c2 === nothing ? θ.W2 * h : θ.W2 * h .+ θ.c2
    n = length(st) ÷ 2
    Shift(st[(n + 1):end]) ∘ Scale(exp.(st[1:n]))
end
function desc(cl::Coupling{<:MLPConditioner{<:CuMatrix{Float32}}}, inv::Bool)
    dm = get!(() -> DeviceMask(cl.mask), MASKS, cl.mask)
    θ = cl.θ
    ptr(c) = c === nothing ? NULLF : pointer(c)
    LayerDesc(COUPLING_MLP, inv, length(dm.idx1), length(dm.idx2), size(θ.W1, 1), θ.act, θ.slope, 0f0,
              pointer(θ.W1), ptr(θ.c1), pointer(θ.W2), ptr(θ.c2), pointer(dm.idx1), pointer(dm.idx2))
end
# The neural spline flow's coupling law (Durkan et al. 2019): the RationalQuadraticSpline of SplineConditioner whose raw
# knots v = W₂*σ.(W₁*x₂ .+ c₁) .+ c₂ come from the hidden layer of MLPConditioner; a callable returning the reference's
# own spline, so the same object also runs on the CPU reference path.  Float32, n1, n2 <= 128, H <= 128, 2 <= K <= 16,
# D <= 1024 on the device; c₁ / c₂ === nothing is a zero shift.
struct MLPSplineConditioner{M<:AbstractMatrix,V1,V2}
    W1::M   # (H × n2)
    c1::V1  # H, or nothing
    W2::M   # ((3K−1)·n1 × H)
    c2::V2  # (3K−1)·n1, or nothing
    K::Int
    B::Float32
    act::Int32      # ACT_TANH or ACT_LEAKY_RELU
    slope::Float32
end
function (θ::MLPSplineConditioner)(x₂)
    u = θ.c1 === nothing ? θ.W1 * x₂ : θ.W1 * x₂ .+ θ.c1
    h = θ.act == ACT_TANH ? tanh.(u) : ifelse.(u .>= 0, u, θ.slope .* u)
    SplineConditioner(θ.W2, θ.c2, θ.K, θ.B)(h)
end
function desc(cl::Coupling{<:MLPSplineConditioner{<:CuMatrix{Float32}}}, inv::Bool)
    dm = get!(() -> DeviceMask(cl.mask), MASKS, cl.mask)
    θ = cl.θ
    ptr(c) = c === nothing ? NULLF : pointer(c)
    LayerDesc(COUPLING_MLP_RQS, inv, length(dm.idx1), length(dm.idx2), size(θ.W1, 1), θ.act | (Int32(θ.K) << 8),
              θ.slope, θ.B, pointer(θ.W1), ptr(θ.c1), pointer(θ.W2), ptr(θ.c2), pointer(dm.idx1), pointer(dm.idx2))
end
# The RealNVP law of MLPConditioner with M >= 2 hidden layers, a Flux Chain(Dense(n2, H, σ), Dense(H, H, σ), …,
# Dense(H, 2n1)): h_1 = σ.(W_in*x₂ .+ c_1), h_l = σ.(W_hid[:, :, l−1]*h_{l−1} .+ c_l), [s; t] = W_out*h_M .+ c_out.  W_hid
# is H × H × (M−1), whose memory order is the packed layout of the descriptor; c packs [c_1; …; c_M; c_out] or is
# `nothing` (no biases at all).  A callable, so the same object also runs on the CPU reference path.  Float32,
# n1, n2 <= 128, H <= 128, M <= 4, D <= 1024 on the device.
struct DeepMLPConditioner{M<:AbstractMatrix,A<:AbstractArray,V}
    W_in::M   # (H × n2)
    W_hid::A  # (H × H × (M−1))
    W_out::M  # (2n1 × H)
    c::V      # M·H + 2n1, or nothing
    act::Int32      # ACT_TANH or ACT_LEAKY_RELU
    slope::Float32
end
function (θ::DeepMLPConditioner)(x₂)
    H, M = size(θ.W_in, 1), size(θ.W_hid, 3) + 1
    σ(v) = θ.act == ACT_TANH ? tanh.(v) : ifelse.(v .>= 0, v, θ.slope .* v)
    bias(l) = θ.c === nothing ? false : θ.c[((l - 1) * H + 1):(l * H)]
    h = σ(θ.W_in * x₂ .+ bias(1))
    for l in 2:M
        h = σ(θ.W_hid[:, :, l - 1] * h .+ bias(l))
    end
    st = θ.c === nothing ? θ.W_out * h : θ.W_out * h .+ θ.c[(M * H + 1):end]
    n = length(st) ÷ 2
    Shift(st[(n + 1):end]) ∘ Scale(exp.(st[1:n]))
end
function desc(cl::Coupling{<:DeepMLPConditioner{<:CuMatrix{Float32}}}, inv::Bool)
    dm = get!(() -> DeviceMask(cl.mask), MASKS, cl.mask)
    θ = cl.θ
    M = size(θ.W_hid, 3) + 1
    LayerDesc(COUPLING_DEEP_MLP, inv, length(dm.idx1), length(dm.idx2), size(θ.W_in, 1), θ.act | (Int32(M) << 8),
              θ.slope, 0f0, pointer(θ.W_in), pointer(θ.W_hid), pointer(θ.W_out), θ.c === nothing ? NULLF : pointer(θ.c),
              pointer(dm.idx1), pointer(dm.idx2))
end
# The neural spline flow's law with the deep network of DeepMLPConditioner: the RationalQuadraticSpline of
# SplineConditioner whose raw knots v = W_out*h_M .+ c_out come from M >= 2 hidden layers.  W_hid is H × H × (M−1) and c
# packs [c_1; …; c_M; c_out] or is `nothing`, as for DeepMLPConditioner.  A callable returning the reference's own spline,
# so the same object also runs on the CPU reference path.  Float32, n1, n2 <= 128, H <= 128, 2 <= K <= 16, M <= 4,
# D <= 1024 on the device.
struct DeepMLPSplineConditioner{M<:AbstractMatrix,A<:AbstractArray,V}
    W_in::M   # (H × n2)
    W_hid::A  # (H × H × (M−1))
    W_out::M  # ((3K−1)·n1 × H)
    c::V      # M·H + (3K−1)·n1, or nothing
    K::Int
    B::Float32
    act::Int32      # ACT_TANH or ACT_LEAKY_RELU
    slope::Float32
end
function (θ::DeepMLPSplineConditioner)(x₂)
    H, M = size(θ.W_in, 1), size(θ.W_hid, 3) + 1
    σ(v) = θ.act == ACT_TANH ? tanh.(v) : ifelse.(v .>= 0, v, θ.slope .* v)
    bias(l) = θ.c === nothing ? false : θ.c[((l - 1) * H + 1):(l * H)]
    h = σ(θ.W_in * x₂ .+ bias(1))
    for l in 2:M
        h = σ(θ.W_hid[:, :, l - 1] * h .+ bias(l))
    end
    SplineConditioner(θ.W_out, θ.c === nothing ? nothing : θ.c[(M * H + 1):end], θ.K, θ.B)(h)
end
function desc(cl::Coupling{<:DeepMLPSplineConditioner{<:CuMatrix{Float32}}}, inv::Bool)
    dm = get!(() -> DeviceMask(cl.mask), MASKS, cl.mask)
    θ = cl.θ
    M = size(θ.W_hid, 3) + 1
    LayerDesc(COUPLING_DEEP_MLP_RQS, inv, length(dm.idx1), length(dm.idx2), size(θ.W_in, 1),
              θ.act | (Int32(θ.K) << 8) | (Int32(M) << 16), θ.slope, θ.B, pointer(θ.W_in), pointer(θ.W_hid),
              pointer(θ.W_out), θ.c === nothing ? NULLF : pointer(θ.c), pointer(dm.idx1), pointer(dm.idx2))
end
desc(cl::Coupling, ::Bool) =
    error("Coupling: only AffineConditioner, SplineConditioner, MLPConditioner, MLPSplineConditioner, " *
          "DeepMLPConditioner and DeepMLPSplineConditioner laws run on the device path (no CPU fallback)")

# Permute(A): y[dst[i]] = x[i] with dst = the row of the single 1 in column i (permute.jl:90-100,152)
const PERMS = IdDict{Any,CuVector{Int32}}()
function desc(b::Permute, inv::Bool)
    dst = get!(PERMS, b) do
        r, c, _ = findnz(b.A)
        d = zeros(Int32, size(b.A, 2)); d[c] .= Int32.(r .- 1)
        cu(d)
    end
    LayerDesc(PERMUTE, inv, 0, 0, 0, 0, 0f0, 0f0, NULLF, NULLF, NULLF, NULLF, pointer(dst), NULLI)
end

# Stacked of elementwise laws on row ranges (stacked.jl:25-59,157-166,242-252): one law code + (a, b) per row
ew_law(::typeof(identity)) = (EW_IDENTITY, 0f0, 0f0)
ew_law(f::Base.Fix1{typeof(broadcast)}) = f.x === exp ? (EW_EXP, 0f0, 0f0) : f.x === log ? (EW_LOG, 0f0, 0f0) :
    f.x === identity ? (EW_IDENTITY, 0f0, 0f0) : error("elementwise($(f.x)) is not on the device path")
ew_law(b::Shift{<:Real}) = (EW_SHIFT, Float32(b.a), 0f0)
ew_law(b::Scale{<:Real}) = (EW_SCALE, Float32(b.a), 0f0)
ew_law(b::LeakyReLU{<:Real}) = (EW_LEAKY_RELU, Float32(b.α), 0f0)
ew_law(b::Logit{<:Real,<:Real}) = (EW_LOGIT, Float32(b.a), Float32(b.b))
ew_law(b::TruncatedBijector{<:Real,<:Real}) = (EW_TRUNCATED, Float32(b.lb), Float32(b.ub))
ew_law(b) = error("Stacked block $(typeof(b)) is not on the device path (no CPU fallback)")
struct DeviceStacked
    code::CuVector{Int32}; a::CuVector{Float32}; b::CuVector{Float32}
end
const STACKS = IdDict{Any,DeviceStacked}()
function DeviceStacked(sb::Stacked)
    D = sb.length_in
    code, a, b = zeros(Int32, D), zeros(Float32, D), zeros(Float32, D)
    for (blk, r) in zip(sb.bs, sb.ranges_in)
        c, pa, pb = ew_law(blk)
        code[r] .= c; a[r] .= pa; b[r] .= pb
    end
    DeviceStacked(cu(code), cu(a), cu(b))
end
function desc(sb::Stacked, inv::Bool)
    ds = get!(() -> DeviceStacked(sb), STACKS, sb)
    LayerDesc(STACKED_EW, inv, 0, 0, 0, 0, 0f0, 0f0, pointer(ds.a), pointer(ds.b), NULLF, NULLF, pointer(ds.code), NULLI)
end
# Scale(A) with a D x D matrix (scale.jl:14,17,35-36): A itself, column-major as CuMatrix stores it; Float32, D <= 256
desc(b::Scale{<:CuMatrix{Float32}}, inv::Bool) =
    LayerDesc(SCALE_MATRIX, inv, 0, 0, 0, 0, 0f0, 0f0, pointer(b.a), NULLF, NULLF, NULLF, NULLI, NULLI)
# Shift / Scale / LeakyReLU with a vector field (shift.jl, scale.jl:16,31-32, leaky_relu.jl:25-29): the law on every row with
# the row's own, trainable parameter, n0 = the law.  Float32 vectors give the descriptor of b2b_chain_run_f32 /
# b2b_chain_vjp_f32; Float64 ones the b2b_layer_desc_f64 of b2b_chain_run_f64 / b2b_chain_vjp_f64 (include/b2b.h).
struct LayerDesc64
    kind::Int32; inverse::Int32
    n0::Int32; n1::Int32; n2::Int32; n3::Int32
    f0::Float64; f1::Float64
    p0::CuPtr{Float64}; p1::CuPtr{Float64}; p2::CuPtr{Float64}; p3::CuPtr{Float64}
    i0::CuPtr{Int32}; i1::CuPtr{Int32}
end
const NULLD = CuPtr{Float64}(0)
const VectorLaw{A} = Union{Shift{<:A},Scale{<:A},LeakyReLU{<:A}}
vec_param(b::Union{Shift,Scale}) = b.a
vec_param(b::LeakyReLU) = b.α
vec_code(::Shift) = EW_SHIFT
vec_code(::Scale) = EW_SCALE
vec_code(::LeakyReLU) = EW_LEAKY_RELU
desc(b::VectorLaw{CuVector{Float32}}, inv::Bool) =
    LayerDesc(ELEMENTWISE_VEC, inv, vec_code(b), 0, 0, 0, 0f0, 0f0, pointer(vec_param(b)), NULLF, NULLF, NULLF, NULLI, NULLI)
desc(b::VectorLaw{CuVector{Float64}}, inv::Bool) =
    LayerDesc64(ELEMENTWISE_VEC, inv, vec_code(b), 0, 0, 0, 0.0, 0.0, pointer(vec_param(b)), NULLD, NULLD, NULLD, NULLI, NULLI)
# Scale(T) with T a LinearAlgebra triangular view of a CuMatrix (scale.jl:14,17,35-36): the parent matrix, column-major, with
# n0 = upper and n1 = unit diagonal; only the triangle is read.  Float32 (D <= 256) or Float64 (D <= 2048).
const TriMat{T} = Union{LowerTriangular{T,<:CuMatrix{T}},UpperTriangular{T,<:CuMatrix{T}},
                        UnitLowerTriangular{T,<:CuMatrix{T}},UnitUpperTriangular{T,<:CuMatrix{T}}}
tri_upper(a) = Int32(a isa Union{UpperTriangular,UnitUpperTriangular})
tri_unit(a) = Int32(a isa Union{UnitLowerTriangular,UnitUpperTriangular})
desc(b::Scale{<:TriMat{Float32}}, inv::Bool) =
    LayerDesc(SCALE_TRIANGULAR, inv, tri_upper(b.a), tri_unit(b.a), 0, 0, 0f0, 0f0, pointer(parent(b.a)), NULLF, NULLF, NULLF,
              NULLI, NULLI)
desc(b::Scale{<:TriMat{Float64}}, inv::Bool) =
    LayerDesc64(SCALE_TRIANGULAR, inv, tri_upper(b.a), tri_unit(b.a), 0, 0, 0.0, 0.0, pointer(parent(b.a)), NULLD, NULLD, NULLD,
                NULLI, NULLI)
# LULinear: the LU-parameterised linear layer y = P·L·U·x, one layer for Permute(p) ∘ Scale(UnitLowerTriangular(factors)) ∘
# Scale(UpperTriangular(factors)).  `factors` packs L (strictly below the diagonal, unit diagonal implied) and U (on and
# above it) as lu(A).factors does, and `p` is lu(A).p (1-based; nothing: the identity), so LULinear(cu(F.factors),
# cu(Int32.(F.p))) of F = lu(A) maps y = A x.  logjac = Σ log|Uᵢᵢ|.  Float32 (D <= 256) or Float64 (D <= 2048); `factors`
# trains as one parameter, both triangles.
struct LULinear{T<:Union{Float32,Float64}} <: Bijectors.Bijector
    factors::CuMatrix{T}
    p::Union{Nothing,CuVector{Int32}}
end
const LU_DST = IdDict{Any,CuVector{Int32}}()  # p .- 1, the descriptor's 0-based destination rows
lu_dst(b::LULinear) = b.p === nothing ? NULLI : pointer(get!(() -> b.p .- Int32(1), LU_DST, b.p))
desc(b::LULinear{Float32}, inv::Bool) =
    LayerDesc(SCALE_LU, inv, 0, 0, 0, 0, 0f0, 0f0, pointer(b.factors), NULLF, NULLF, NULLF, lu_dst(b), NULLI)
desc(b::LULinear{Float64}, inv::Bool) =
    LayerDesc64(SCALE_LU, inv, 0, 0, 0, 0, 0.0, 0.0, pointer(b.factors), NULLD, NULLD, NULLD, lu_dst(b), NULLI)
# MaskedAutoregressive: MAF / IAF's affine layer with a MADE conditioner, y = x .* exp.(s) .+ t with
# [s; t] = (M₂ .* W2) * σ.((M₁ .* W1) * x .+ c1) .+ c2, masks M₁[k, r] = (r <= m_k), M₂[i, k] = M₂[D+i, k] = (m_k < i) from
# the hidden units' integer degrees m (so sᵢ, tᵢ depend on x₁..x_{i−1} only); logjac = Σ s.  W1 is (H × D), W2 (2D × H),
# c1 / c2 === nothing is a zero shift, σ = tanh or LeakyReLU(slope).  The inverse recovers x row by row; MAF is a chain of
# inverse(layer)s.  Float32, D <= 128, H <= 256 on the device; the same object runs on the CPU reference path.
struct MaskedAutoregressive{M<:AbstractMatrix,V1,V2,I<:AbstractVector} <: Bijectors.Bijector
    W1::M   # (H × D)
    c1::V1  # H, or nothing
    W2::M   # (2D × H)
    c2::V2  # 2D, or nothing
    degrees::I      # m (Int32 on the device)
    act::Int32      # ACT_TANH or ACT_LEAKY_RELU
    slope::Float32
end
function ar_shift_scale(b::MaskedAutoregressive, X::AbstractMatrix)
    D, m = size(X, 1), collect(b.degrees)
    W1 = ifelse.((1:D)' .<= m, b.W1, zero(eltype(b.W1)))  # entries outside the masks are never used
    W2 = ifelse.(repeat(m' .< (1:D), 2, 1), b.W2, zero(eltype(b.W2)))
    u = b.c1 === nothing ? W1 * X : W1 * X .+ b.c1
    h = b.act == ACT_TANH ? tanh.(u) : ifelse.(u .>= 0, u, b.slope .* u)
    st = b.c2 === nothing ? W2 * h : W2 * h .+ b.c2
    return st[1:D, :], st[(D + 1):end, :]
end
function with_logabsdet_jacobian(b::MaskedAutoregressive, x::AbstractVecOrMat)
    X = x isa AbstractVector ? reshape(x, :, 1) : x
    s, t = ar_shift_scale(b, X)
    Y, lj = X .* exp.(s) .+ t, vec(sum(s; dims=1))
    return x isa AbstractVector ? (vec(Y), lj[1]) : (Y, lj)
end
function with_logabsdet_jacobian(ib::Inverse{<:MaskedAutoregressive}, y::AbstractVecOrMat)
    Y = y isa AbstractVector ? reshape(y, :, 1) : y
    X = zero(Y)
    for i in axes(Y, 1)  # rows >= i of X are still 0 and do not reach sᵢ, tᵢ
        s, t = ar_shift_scale(ib.orig, X)
        X[i:i, :] .= (Y[i:i, :] .- t[i:i, :]) ./ exp.(s[i:i, :])
    end
    lj = -vec(sum(first(ar_shift_scale(ib.orig, X)); dims=1))
    return y isa AbstractVector ? (vec(X), lj[1]) : (X, lj)
end
transform(b::Union{MaskedAutoregressive,Inverse{<:MaskedAutoregressive}}, x::AbstractVecOrMat) =
    first(with_logabsdet_jacobian(b, x))
function desc(b::MaskedAutoregressive{<:CuMatrix{Float32}}, inv::Bool)
    ptr(c) = c === nothing ? NULLF : pointer(c)
    LayerDesc(AUTOREGRESSIVE_MLP, inv, 0, 0, size(b.W1, 1), b.act, b.slope, 0f0, pointer(b.W1), ptr(b.c1), pointer(b.W2),
              ptr(b.c2), pointer(b.degrees), NULLI)
end
# a whole-column elementwise law is a one-block Stacked
const ElementwiseLaw = Union{Shift{<:Real},Scale{<:Real},LeakyReLU{<:Real},Logit{<:Real,<:Real},TruncatedBijector{<:Real,<:Real}}

# ---- chains: Base.ComposedFunction trees are flattened inner-most first ------------------------------
flatten(f::ComposedFunction) = (flatten(f.inner)..., flatten(f.outer)...)
flatten(f) = (f,)
descs(f, inv::Bool) = inv ? [desc(b, true) for b in reverse(flatten(f))] : [desc(b, false) for b in flatten(f)]

const DeviceLayer = Union{PlanarLayer{<:CuVector{Float32}},RadialLayer{<:CuVector{Float32}},
                          RationalQuadraticSpline{<:CuMatrix{Float32}},InvertibleBatchNorm{<:CuVector{Float32}},
                          Coupling{<:AffineConditioner},Coupling{<:SplineConditioner{<:CuMatrix{Float32}}},
                          Coupling{<:MLPConditioner{<:CuMatrix{Float32}}},Coupling{<:MLPSplineConditioner{<:CuMatrix{Float32}}},
                          Coupling{<:DeepMLPConditioner{<:CuMatrix{Float32}}},
                          Coupling{<:DeepMLPSplineConditioner{<:CuMatrix{Float32}}},
                          Scale{<:CuMatrix{Float32}},Scale{<:TriMat{Float32}},LULinear{Float32},VectorLaw{CuVector{Float32}},Permute,
                          MaskedAutoregressive{<:CuMatrix{Float32},<:Any,<:Any,<:CuVector{Int32}},
                          Stacked}
const DeviceLeaf = Union{DeviceLayer,Inverse{<:DeviceLayer}}
is_device(f::ComposedFunction) = is_device(f.inner) && is_device(f.outer)
is_device(::DeviceLeaf) = true
is_device(_) = false

function run_chain(ds::Vector{LayerDesc}, x::CuMatrix{Float32}; y=similar(x), logjac=CUDA.zeros(Float32, size(x, 2)),
                   sum_out=nothing, accumulate=false)
    D, N = size(x)
    ws_bytes = ccall((:b2b_chain_workspace_bytes, libb2b), Csize_t,
                     (Ptr{LayerDesc}, Int32, Int32, Int64, Cint, Cint), ds, length(ds), D, N, y !== nothing, sum_out !== nothing)
    ws = CuVector{UInt8}(undef, ws_bytes)
    GC.@preserve ds ws begin
        check(ccall((:b2b_chain_run_f32, libb2b), Cint,
            (Ptr{LayerDesc}, Int32, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float64},
             Int32, Int64, Int64, Int64, Cint, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
            ds, length(ds), pointer(x), y === nothing ? NULLF : pointer(y),
            logjac === nothing ? NULLF : pointer(logjac),
            sum_out === nothing ? CuPtr{Float64}(0) : pointer(sum_out),
            D, N, stride(x, 2), y === nothing ? D : stride(y, 2), accumulate, pointer(ws), ws_bytes, stream_handle()))
    end
    return y, logjac
end

# ---- the methods Bijectors.jl dispatches to ------------------------------------------------------------
# Leaves: Bijectors' own layer types with CuArray parameters (and Inverse of them).
with_logabsdet_jacobian(b::DeviceLeaf, x::CuMatrix{Float32}) = run_chain(descs(b, false), x)
transform(b::DeviceLeaf, x::CuMatrix{Float32}) = first(run_chain(descs(b, false), x; logjac=nothing))
logabsdetjac(b::DeviceLeaf, x::CuMatrix{Float32}) = last(run_chain(descs(b, false), x; y=nothing))

# InvertibleBatchNorm on arrays of more than two dimensions (normalise.jl:41-47: channel axis ndims − 1, batch axis last):
# the slab of one batch element is a column of S·C numbers whose row s + S·c belongs to channel c, so the elementwise map
# is the D×N kernel on a reshape of the same memory with every channel's parameters repeated S times; the log-Jacobian
# the reference returns has no factor S (:66) -- it is the C-channel layer's own, evaluated on a C×B batch.
const DeviceBN = InvertibleBatchNorm{<:CuVector{Float32}}
function batchnorm_nd(b::Union{DeviceBN,Inverse{<:DeviceBN}}, x::CuArray{Float32})
    bn = b isa Inverse ? b.orig : b
    C, B = size(x, ndims(x) - 1), size(x, ndims(x))
    C == length(bn.b) || error("InvertibleBatchNorm expected $(length(bn.b)) channels, got $C")
    S = div(length(x), C * B)
    wide = InvertibleBatchNorm(repeat(bn.b; inner=S), repeat(bn.logs; inner=S), repeat(bn.m; inner=S),
                               repeat(bn.v; inner=S), bn.eps, bn.mtm)
    y = first(run_chain(descs(b isa Inverse ? inverse(wide) : wide, false), reshape(x, S * C, B); logjac=nothing))
    logjac = last(run_chain(descs(b, false), CUDA.zeros(Float32, C, B); y=nothing))
    return reshape(y, size(x)), logjac
end
with_logabsdet_jacobian(b::Union{DeviceBN,Inverse{<:DeviceBN}}, x::CuArray{Float32,3}) = batchnorm_nd(b, x)
with_logabsdet_jacobian(b::Union{DeviceBN,Inverse{<:DeviceBN}}, x::CuArray{Float32,4}) = batchnorm_nd(b, x)
with_logabsdet_jacobian(b::Union{DeviceBN,Inverse{<:DeviceBN}}, x::CuArray{Float32,5}) = batchnorm_nd(b, x)

# Host-resident PlanarLayer chains (fields are plain Arrays) on a device batch: parameters travel as kernel arguments.
const HostPlanar = PlanarLayer{<:Vector{Float32}}
all_host_planar(f) = all(b -> b isa HostPlanar, flatten(f))
function planar_hostparams(f, x::CuMatrix{Float32}; inv::Bool=false)
    ls = inv ? reverse(collect(flatten(f))) : collect(flatten(f))
    w, u, b = reduce(hcat, [l.w for l in ls]), reduce(hcat, [l.u for l in ls]), Float32[first(l.b) for l in ls]
    y, logjac = similar(x), CUDA.zeros(Float32, size(x, 2))
    check(ccall((:b2b_planar_chain_hostparams_f32, libb2b), Cint,
        (Ptr{Float32}, Ptr{Float32}, Ptr{Float32}, Int32, Cint, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         Int32, Int64, Int64, Int64, Cint, Ptr{Cvoid}),
        w, u, b, length(ls), inv, pointer(x), pointer(y), pointer(logjac),
        size(x, 1), size(x, 2), stride(x, 2), stride(y, 2), false, stream_handle()))
    return y, logjac
end
with_logabsdet_jacobian(b::HostPlanar, x::CuMatrix{Float32}) = planar_hostparams(b, x)

# ∘-chains: ONE method per generic function (no ambiguity).  It takes the chain only when every leaf is a device layer
# (or every leaf a host-resident PlanarLayer); anything else goes back to the reference's own generic method
# (ChangesOfVariables' rule for ComposedFunction), so compositions of unrelated functions on a CuMatrix are untouched.
function with_logabsdet_jacobian(f::ComposedFunction, x::CuMatrix{Float32})
    is_device(f) && return run_chain(descs(f, false), x)
    all_host_planar(f) && return planar_hostparams(f, x)
    return invoke(with_logabsdet_jacobian, Tuple{ComposedFunction,Any}, f, x)
end
function transform(f::ComposedFunction, x::CuMatrix{Float32})
    is_device(f) && return first(run_chain(descs(f, false), x; logjac=nothing))
    return invoke(transform, Tuple{ComposedFunction,Any}, f, x)
end
function logabsdetjac(f::ComposedFunction, x::CuMatrix{Float32})
    is_device(f) && return last(run_chain(descs(f, false), x; y=nothing))
    return invoke(logabsdetjac, Tuple{ComposedFunction,Any}, f, x)
end
# in-place variants (src/interface.jl:175-176, 212-218): y may alias x, logjac accumulates
function Bijectors.with_logabsdet_jacobian!(b::Union{DeviceLeaf,ComposedFunction}, x::CuMatrix{Float32},
                                            y::CuMatrix{Float32}, logjac::CuVector{Float32})
    is_device(b) || error("with_logabsdet_jacobian!: not a device chain")
    run_chain(descs(b, false), x; y=y, logjac=logjac, accumulate=true)
end

# Training-mode InvertibleBatchNorm (normalise.jl:51-60): batch statistics (over all ranks when `comm` is given), moving
# statistics updated in place.  The reference's global istraining() switch is this separate entry point.
function batchnorm_train!(bn::InvertibleBatchNorm{<:CuVector{Float32}}, x::CuMatrix{Float32}; comm=nothing)
    D, N = size(x)
    y, logjac = similar(x), CUDA.zeros(Float32, N)
    nbytes = ccall((:b2b_batchnorm_train_workspace_bytes, libb2b), Csize_t, (Int32,), D)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve ws check(ccall((:b2b_batchnorm_train_fwd_f32, libb2b), Cint,
        (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         Cfloat, Cfloat, Int32, Int64, Int64, Int64, Cint, Ptr{Cvoid}, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        pointer(x), pointer(y), pointer(logjac), pointer(bn.b), pointer(bn.logs), pointer(bn.m), pointer(bn.v),
        Float32(bn.eps), Float32(bn.mtm), D, N, stride(x, 2), stride(y, 2), false,
        comm === nothing ? C_NULL : comm.handle, pointer(ws), nbytes, stream_handle()))
    return y, logjac
end

# Its reverse mode: cotangents of x (through the batch statistics, over all ranks when `comm` is given) and of b, logs
# (summed over this rank's columns).  The moving statistics are not touched.
function batchnorm_train_vjp(bn::InvertibleBatchNorm{<:CuVector{Float32}}, x::CuMatrix{Float32}, ȳ::CuMatrix{Float32},
                             l̄::CuVector{Float32}; comm=nothing)
    D, N = size(x)
    x̄ = similar(x); b̄ = CUDA.zeros(Float32, D); l̄ogs = CUDA.zeros(Float32, D)
    nbytes = ccall((:b2b_batchnorm_train_vjp_workspace_bytes, libb2b), Csize_t, (Int32,), D)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve ws check(ccall((:b2b_batchnorm_train_vjp_f32, libb2b), Cint,
        (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         Cfloat, Int32, Int64, Int64, Int64, Int64, Ptr{Cvoid}, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        pointer(x), pointer(ȳ), pointer(l̄), pointer(x̄), pointer(b̄), pointer(l̄ogs), pointer(bn.logs),
        Float32(bn.eps), D, N, stride(x, 2), stride(ȳ, 2), stride(x̄, 2),
        comm === nothing ? C_NULL : comm.handle, pointer(ws), nbytes, stream_handle()))
    return x̄, b̄, l̄ogs
end

# Reverse mode: a ChainRulesCore.rrule for device planar chains (what ext/BijectorsChainRulesCoreExt.jl does for the CPU
# path, incl. the implicit find_alpha rule :42-46).  ȳ, l̄ are the cotangents of (y, logjac).
function planar_chain_vjp(f, x::CuMatrix{Float32}, ȳ::CuMatrix{Float32}, l̄::CuVector{Float32}; inv::Bool=false)
    ds = descs(f, inv)
    L, (D, N) = length(ds), size(x)
    x̄ = similar(x); w̄ = CUDA.zeros(Float32, D, L); ū = CUDA.zeros(Float32, D, L); b̄ = CUDA.zeros(Float32, L)
    nbytes = ccall((:b2b_planar_chain_vjp_workspace_bytes, libb2b), Csize_t, (Int32, Int32, Int64), L, D, N)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve ds ws check(ccall((:b2b_planar_chain_vjp_f32, libb2b), Cint,
        (Ptr{LayerDesc}, Int32, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         CuPtr{Float32}, CuPtr{Float32}, Int32, Int64, Int64, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        ds, L, pointer(x), pointer(ȳ), pointer(l̄), pointer(x̄), pointer(w̄), pointer(ū), pointer(b̄),
        D, N, stride(x, 2), stride(ȳ, 2), stride(x̄, 2), pointer(ws), nbytes, stream_handle()))
    return x̄, w̄, ū, b̄        # column l of w̄ / ū and b̄[l] belong to the l-th applied layer
end

function radial_chain_vjp(f, x::CuMatrix{Float32}, ȳ::CuMatrix{Float32}, l̄::CuVector{Float32})
    ds = descs(f, false)
    L, (D, N) = length(ds), size(x)
    x̄ = similar(x); ᾱ = CUDA.zeros(Float32, L); β̄ = CUDA.zeros(Float32, L); z̄0 = CUDA.zeros(Float32, D, L)
    nbytes = ccall((:b2b_radial_chain_vjp_workspace_bytes, libb2b), Csize_t, (Int32, Int32), L, D)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve ds ws check(ccall((:b2b_radial_chain_vjp_f32, libb2b), Cint,
        (Ptr{LayerDesc}, Int32, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         CuPtr{Float32}, CuPtr{Float32}, Int32, Int64, Int64, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        ds, L, pointer(x), pointer(ȳ), pointer(l̄), pointer(x̄), pointer(ᾱ), pointer(β̄), pointer(z̄0),
        D, N, stride(x, 2), stride(ȳ, 2), stride(x̄, 2), pointer(ws), nbytes, stream_handle()))
    return x̄, ᾱ, β̄, z̄0        # cotangents of the raw fields α_, β, z_0 of each layer
end

# Reverse mode of the RealNVP layer kinds: one affine Coupling (incl. the `combine` pullback,
# ext/BijectorsChainRulesCoreExt.jl:48-62) / one eval-mode InvertibleBatchNorm, either direction.
function coupling_vjp(cl, x::CuMatrix{Float32}, ȳ::CuMatrix{Float32}, l̄::CuVector{Float32}; inv::Bool=false)
    d = [desc(cl, inv)]
    n1, n2, (D, N) = Int(d[1].n0), Int(d[1].n1), size(x)
    x̄ = similar(x); W̄ = CUDA.zeros(Float32, 2n1, n2); c̄ = CUDA.zeros(Float32, 2n1)
    nbytes = ccall((:b2b_coupling_affine_vjp_workspace_bytes, libb2b), Csize_t, (Int32, Int32), n1, n2)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve d ws check(ccall((:b2b_coupling_affine_vjp_f32, libb2b), Cint,
        (Ptr{LayerDesc}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         Int32, Int64, Int64, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        d, pointer(x), pointer(ȳ), pointer(l̄), pointer(x̄), pointer(W̄), pointer(c̄),
        D, N, stride(x, 2), stride(ȳ, 2), stride(x̄, 2), pointer(ws), nbytes, stream_handle()))
    return x̄, W̄, c̄
end
function batchnorm_vjp(bn, x::CuMatrix{Float32}, ȳ::CuMatrix{Float32}, l̄::CuVector{Float32}; inv::Bool=false)
    d = [desc(bn, inv)]
    D, N = size(x)
    x̄ = similar(x); b̄ = CUDA.zeros(Float32, D); l̄ogs = CUDA.zeros(Float32, D)
    nbytes = ccall((:b2b_batchnorm_eval_vjp_workspace_bytes, libb2b), Csize_t, (Int32,), D)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve d ws check(ccall((:b2b_batchnorm_eval_vjp_f32, libb2b), Cint,
        (Ptr{LayerDesc}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         Int32, Int64, Int64, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        d, pointer(x), pointer(ȳ), pointer(l̄), pointer(x̄), pointer(b̄), pointer(l̄ogs),
        D, N, stride(x, 2), stride(ȳ, 2), stride(x̄, 2), pointer(ws), nbytes, stream_handle()))
    return x̄, b̄, l̄ogs
end

# Reverse mode of one RationalQuadraticSpline (either direction): cotangents of the input and of the processed fields
# widths / heights / derivatives (D × K+1 each, like the fields themselves).
function rqs_vjp(b, x::CuMatrix{Float32}, ȳ::CuMatrix{Float32}, l̄::CuVector{Float32}; inv::Bool=false)
    d = [desc(b, inv)]
    K1, (D, N) = Int(d[1].n0), size(x)
    x̄ = similar(x); W̄ = CUDA.zeros(Float32, D, K1); H̄ = CUDA.zeros(Float32, D, K1); D̄ = CUDA.zeros(Float32, D, K1)
    nbytes = ccall((:b2b_rqs_vjp_workspace_bytes, libb2b), Csize_t, (Int32, Int32), K1, D)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve d ws check(ccall((:b2b_rqs_vjp_f32, libb2b), Cint,
        (Ptr{LayerDesc}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
         CuPtr{Float32}, Int32, Int64, Int64, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        d, pointer(x), pointer(ȳ), pointer(l̄), pointer(x̄), pointer(W̄), pointer(H̄), pointer(D̄),
        D, N, stride(x, 2), stride(ȳ, 2), stride(x̄, 2), pointer(ws), nbytes, stream_handle()))
    return x̄, W̄, H̄, D̄
end

# Reverse mode of ANY device chain (b2b_chain_vjp_f32): `f` (or inverse(f) with inv=true); ȳ, l̄ the cotangents of
# (y, logjac), `nothing` = zeros.  Returns x̄ and, per descriptor in application order, the cotangents of its trainable
# fields (PlanarLayer w u b, RadialLayer α_ β z_0, RQS widths heights derivatives, Coupling W c, Scale(A) a, vector Shift /
# Scale a and LeakyReLU α, BatchNorm b logs, the
# terminal MvNormal's μ σ) in the fields' shapes; `nothing` for fields without one.
# Hidden units H, spline bins K and hidden layers M of a coupling descriptor (0 where the kind has none), decoded here only:
# n2 is K or H, and n3 packs σ | K << 8, σ | M << 8 or σ | K << 8 | M << 16 (include/b2b.h).
coupling_hkm(d::LayerDesc) =
    d.kind == COUPLING_RQS ? (0, Int(d.n2), 0) : d.kind == COUPLING_MLP ? (Int(d.n2), 0, 1) :
    d.kind == COUPLING_MLP_RQS ? (Int(d.n2), Int(d.n3 >> 8), 1) :
    d.kind == COUPLING_DEEP_MLP ? (Int(d.n2), 0, Int(d.n3 >> 8)) :
    d.kind == COUPLING_DEEP_MLP_RQS ? (Int(d.n2), Int((d.n3 >> 8) & 255), Int(d.n3 >> 16)) : (0, 0, 0)
function vjp_slots(d::LayerDesc, D::Integer)
    z(dims...) = CUDA.zeros(Float32, dims...)
    d.kind == PLANAR && return (z(D), z(D), z(1))
    d.kind == RADIAL && return (z(1), z(1), z(D))
    d.kind == RQS && return (z(D, d.n0), z(D, d.n0), z(D, d.n0))
    if d.kind in (COUPLING_AFFINE, COUPLING_RQS, COUPLING_MLP, COUPLING_MLP_RQS, COUPLING_DEEP_MLP, COUPLING_DEEP_MLP_RQS)
        H, K, M = coupling_hkm(d)
        J = K > 0 ? (3K - 1) * d.n0 : 2d.n0  # rows of the last layer
        H == 0 && return (z(J, d.n1), d.p1 == NULLF ? nothing : z(J))
        d.kind in (COUPLING_DEEP_MLP, COUPLING_DEEP_MLP_RQS) &&
            return (z(H, d.n1), z(H, H, M - 1), z(J, H), d.p3 == NULLF ? nothing : z(M * H + J))
        return (z(H, d.n1), d.p1 == NULLF ? nothing : z(H), z(J, H), d.p3 == NULLF ? nothing : z(J))
    end
    d.kind == SCALE_MATRIX && return (z(D, D),)
    d.kind == SCALE_TRIANGULAR && return (z(D, D),)  # exactly 0 outside the triangle; leaf_tangent wraps it
    d.kind == SCALE_LU && return (z(D, D),)
    d.kind == AUTOREGRESSIVE_MLP &&
        return (z(d.n2, D), d.p1 == NULLF ? nothing : z(d.n2), z(2D, d.n2), d.p3 == NULLF ? nothing : z(2D))  # factors̄, packed as factors: L̄ below the diagonal, Ū on and above it
    d.kind == ELEMENTWISE_VEC && return (z(D),)  # Shift / Scale a, LeakyReLU α
    d.kind == BATCHNORM && return (z(D), z(D))
    d.kind == MVNORMAL_DIAG && return (d.p0 == NULLF ? nothing : z(D), d.p1 == NULLF ? nothing : z(D))
    d.kind == MVNORMAL_TRIL && return (d.p0 == NULLF ? nothing : z(D), z(D, D))
    return ()
end
chain_vjp(f, x::CuMatrix{Float32}, ȳ, l̄; inv::Bool=false) = chain_vjp(descs(f, inv), x, ȳ, l̄)
function chain_vjp(ds::Vector{LayerDesc}, x::CuMatrix{Float32}, ȳ, l̄)
    L, (D, N) = length(ds), size(x)
    bars = [vjp_slots(d, D) for d in ds]
    ptrs = Ptr{Cvoid}[i <= length(b) && b[i] !== nothing ? Ptr{Cvoid}(UInt(pointer(b[i]))) : C_NULL for b in bars for i in 1:4]
    x̄ = similar(x)
    nbytes = ccall((:b2b_chain_vjp_workspace_bytes, libb2b), Csize_t, (Ptr{LayerDesc}, Int32, Int32, Int64), ds, L, D, N)
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve ds bars ptrs ws ȳ l̄ check(ccall((:b2b_chain_vjp_f32, libb2b), Cint,
        (Ptr{LayerDesc}, Int32, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Ptr{Ptr{Cvoid}}, Int32,
         Int64, Int64, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        ds, L, pointer(x), ȳ === nothing ? NULLF : pointer(ȳ), l̄ === nothing ? NULLF : pointer(l̄), pointer(x̄), ptrs,
        D, N, stride(x, 2), ȳ === nothing ? D : stride(ȳ, 2), stride(x̄, 2), pointer(ws), nbytes, stream_handle()))
    return x̄, bars
end
# The base distribution as the terminal descriptor, with the device arrays it points to (keep them alive while it is
# used).  The covariance type decides the op: a diagonal one (PDiagMat, ScalMat) is MVNORMAL_DIAG with σ = sqrt.(var(d)),
# a dense PDMat (FullNormal) is MVNORMAL_TRIL with its Cholesky factor L.  Any other covariance type has no device op.
function base_desc(d::MvNormal)
    μ, Σ = cu(Float32.(mean(d))), d.Σ
    if Σ isa PDiagMat || Σ isa ScalMat
        σ = cu(Float32.(sqrt.(var(d))))
        return LayerDesc(MVNORMAL_DIAG, 0, 0, 0, 0, 0, 0f0, 0f0, pointer(μ), pointer(σ), NULLF, NULLF, NULLI, NULLI), (μ, σ)
    elseif Σ isa PDMat
        L = cu(Matrix{Float32}(cholesky(Σ).L))   # column-major, lower triangle
        return LayerDesc(MVNORMAL_TRIL, 0, 0, 0, 0, 0, 0f0, 0f0, pointer(μ), pointer(L), NULLF, NULLF, NULLI, NULLI), (μ, L)
    end
    error("B200Bijectors: no device path for an MvNormal with covariance of type $(typeof(Σ)) " *
          "(PDiagMat, ScalMat and PDMat are supported)")
end

# Reverse mode of logpdf(td, y) with cotangent l̄ of the logpdf vector: (ȳ, flow cotangents in flow order, base
# cotangents: (μ̄, σ̄) for a diagonal covariance, (μ̄, L̄) with L̄ lower triangular for a PDMat).
function logpdf_vjp(td::TransformedDistribution{<:MvNormal}, y::CuMatrix{Float32}, l̄::CuVector{Float32})
    ds = descs(td.transform, true)
    term, keep = base_desc(td.dist)
    push!(ds, term)
    ȳ, bars = GC.@preserve keep chain_vjp(ds, y, nothing, l̄)
    return ȳ, reverse(bars[1:end-1]), bars[end]
end

# rand(rng, td, n) (src/transformed_distribution.jl:212-224): the base samples are generated INSIDE the chain kernel
# (Philox4x32-10 + Box-Muller); `seed` plays the role of rng, `column_offset` continues one stream across column shards.
function device_rand(td::TransformedDistribution{<:MvNormal}, n::Integer; seed::UInt64=rand(UInt64), offset::UInt64=UInt64(0),
                     column_offset::Integer=0)
    ds = descs(td.transform, false)
    D = length(td.dist)
    term, keep = base_desc(td.dist)
    y = CuMatrix{Float32}(undef, D, n)
    ws_bytes = ccall((:b2b_chain_workspace_bytes, libb2b), Csize_t,
                     (Ptr{LayerDesc}, Int32, Int32, Int64, Cint, Cint), ds, length(ds), D, n, true, false)
    ws = CuVector{UInt8}(undef, ws_bytes)
    # y = μ + σ .* z (diagonal) or μ + L z (PDMat), z from the same Philox stream
    if term.kind == MVNORMAL_TRIL
        GC.@preserve ds keep ws check(ccall((:b2b_chain_sample_tril_f32, libb2b), Cint,
            (Ptr{LayerDesc}, Int32, CuPtr{Float32}, CuPtr{Float32}, UInt64, UInt64, Int64, CuPtr{Float32}, CuPtr{Float32},
             Int32, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
            ds, length(ds), term.p0, term.p1, seed, offset, column_offset, pointer(y), NULLF,
            D, n, stride(y, 2), pointer(ws), ws_bytes, stream_handle()))
    else
        GC.@preserve ds keep ws check(ccall((:b2b_chain_sample_f32, libb2b), Cint,
            (Ptr{LayerDesc}, Int32, CuPtr{Float32}, CuPtr{Float32}, UInt64, UInt64, Int64, CuPtr{Float32}, CuPtr{Float32},
             Int32, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
            ds, length(ds), term.p0, term.p1, seed, offset, column_offset, pointer(y), NULLF,
            D, n, stride(y, 2), pointer(ws), ws_bytes, stream_handle()))
    end
    return y
end

# Reparameterised sampling (variational inference, docs/src/advi.md; the reference keeps non-in-place rand for
# "differentiating sampling wrt. params of `td.dist` or params of `Bijector`", src/transformed_distribution.jl:210-213).
# rand_logpdf: the samples device_rand draws (bit for bit) and their log-density log q(y) in the same pass.
function rand_logpdf(td::TransformedDistribution{<:MvNormal}, n::Integer; seed::UInt64=rand(UInt64),
                     offset::UInt64=UInt64(0), column_offset::Integer=0)
    ds = descs(td.transform, false)
    D, L = length(td.dist), length(ds)
    base, keep = base_desc(td.dist)
    bd = [base]
    y = CuMatrix{Float32}(undef, D, n)
    lq = CuVector{Float32}(undef, n)
    nbytes = ccall((:b2b_chain_sample_logq_workspace_bytes, libb2b), Csize_t,
                   (Ptr{LayerDesc}, Int32, Ptr{LayerDesc}, Int32, Int64), ds, L, bd, D, n)
    nbytes == 0 && error("B200Bijectors: rand_logpdf: the device path refuses this flow and base")
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve ds bd keep ws check(ccall((:b2b_chain_sample_logq_f32, libb2b), Cint,
        (Ptr{LayerDesc}, Int32, Ptr{LayerDesc}, UInt64, UInt64, Int64, CuPtr{Float32}, CuPtr{Float32}, Int32, Int64, Int64,
         CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        ds, L, bd, seed, offset, column_offset, pointer(y), pointer(lq), D, n, stride(y, 2), pointer(ws), nbytes,
        stream_handle()))
    return y, lq
end

# Reverse mode of rand_logpdf with the draw held fixed: ȳ, q̄ the cotangents of (y, log q), `nothing` = zeros.  Returns
# the flow's cotangents per descriptor in application order (the fields of chain_vjp) and the base's (μ̄, σ̄) or
# (μ̄, L̄), L̄ lower triangular; all summed over the n columns.
function rand_vjp(td::TransformedDistribution{<:MvNormal}, n::Integer, ȳ, q̄; seed::UInt64,
                  offset::UInt64=UInt64(0), column_offset::Integer=0)
    ds = descs(td.transform, false)
    D, L = length(td.dist), length(ds)
    base, keep = base_desc(td.dist)
    bd = [base]
    bars = [vjp_slots(d, D) for d in vcat(ds, bd)]
    ptrs = Ptr{Cvoid}[i <= length(b) && b[i] !== nothing ? Ptr{Cvoid}(UInt(pointer(b[i]))) : C_NULL for b in bars for i in 1:4]
    nbytes = ccall((:b2b_chain_sample_vjp_workspace_bytes, libb2b), Csize_t,
                   (Ptr{LayerDesc}, Int32, Ptr{LayerDesc}, Int32, Int64), ds, L, bd, D, n)
    nbytes == 0 && error("B200Bijectors: rand_vjp: the device path refuses this flow and base")
    ws = CuVector{UInt8}(undef, nbytes)
    GC.@preserve ds bd keep bars ptrs ws ȳ q̄ check(ccall((:b2b_chain_sample_vjp_f32, libb2b), Cint,
        (Ptr{LayerDesc}, Int32, Ptr{LayerDesc}, UInt64, UInt64, Int64, CuPtr{Float32}, Int64, CuPtr{Float32},
         Ptr{Ptr{Cvoid}}, Int32, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        ds, L, bd, seed, offset, column_offset, ȳ === nothing ? NULLF : pointer(ȳ), ȳ === nothing ? D : stride(ȳ, 2),
        q̄ === nothing ? NULLF : pointer(q̄), ptrs, D, n, pointer(ws), nbytes, stream_handle()))
    return bars[1:end-1], bars[end]
end

# Structural tangents of what rand_vjp returns.  The transform: flatten() lists the leaves inner-most first, one
# descriptor each, so a ComposedFunction takes its inner part's cotangents first.  A leaf's trainable fields are the first
# fields of its struct in slot order (PlanarLayer w u b, RadialLayer α_ β z_0, RationalQuadraticSpline widths heights
# derivatives, InvertibleBatchNorm b logs, Scale a, vector Shift a and LeakyReLU α), a Coupling's those of its conditioner θ, and Inverse wraps `orig`.
function transform_tangent(f, bars, k::Base.RefValue{Int})
    f isa ComposedFunction || return leaf_tangent(f, bars[k[] += 1])
    inner = transform_tangent(f.inner, bars, k)
    return ChainRulesCore.Tangent{typeof(f)}(outer=transform_tangent(f.outer, bars, k), inner=inner)
end
function leaf_tangent(b, bar)
    all(t -> t === nothing, bar) && return NoTangent()
    b isa Inverse && return ChainRulesCore.Tangent{typeof(b)}(orig=leaf_tangent(b.orig, bar))
    b isa Coupling && return ChainRulesCore.Tangent{typeof(b)}(θ=leaf_tangent(b.θ, bar))
    names = fieldnames(typeof(b))
    return ChainRulesCore.Tangent{typeof(b)}(; (names[i] => bar[i] for i in eachindex(bar) if bar[i] !== nothing)...)
end
# LULinear: factors̄ only (the permutation has no cotangent)
leaf_tangent(b::LULinear, bar) = bar[1] === nothing ? NoTangent() : ChainRulesCore.Tangent{typeof(b)}(factors=bar[1])
# MaskedAutoregressive: W̄1 c̄1 W̄2 c̄2 (c̄ only where the layer has c), W̄ exactly 0 outside the masks
leaf_tangent(b::MaskedAutoregressive, bar) = all(t -> t === nothing, bar) ? NoTangent() :
    ChainRulesCore.Tangent{typeof(b)}(; (k => v for (k, v) in zip((:W1, :c1, :W2, :c2), bar) if v !== nothing)...)
# a triangular Scale's T̄ in the triangular type of its field
leaf_tangent(b::Scale{<:TriMat}, bar) =
    bar[1] === nothing ? NoTangent() : ChainRulesCore.Tangent{typeof(b)}(a=Base.typename(typeof(b.a)).wrapper(bar[1]))
# The base: μ̄, and the covariance's tangent from σ̄ or L̄ (Σ = diag(σ²): Σ̄ᵢᵢ = σ̄ᵢ/(2σᵢ); Σ = L Lᵀ: Σ̄ = sym(L⁻ᵀ Φ(Lᵀ L̄) L⁻¹)/2,
# Φ the lower triangle with its diagonal halved).
function base_tangent(d::MvNormal, (μ̄, p̄))
    Σ = d.Σ
    if Σ isa PDMat
        L = Matrix(cholesky(Σ).L)
        P = LowerTriangular(L' * Array(p̄))
        P[diagind(P)] ./= 2
        S = L' \ (Matrix(P) / L)
        Σ̄ = ChainRulesCore.Tangent{typeof(Σ)}(mat=(S + S') / 2)
    else
        g = Array(p̄) ./ (2 .* sqrt.(var(d)))
        Σ̄ = Σ isa ScalMat ? ChainRulesCore.Tangent{typeof(Σ)}(value=sum(g)) : ChainRulesCore.Tangent{typeof(Σ)}(diag=g)
    end
    return ChainRulesCore.Tangent{typeof(d)}(μ=Array(μ̄), Σ=Σ̄)
end

# The ELBO's gradient through the sampler: the pullback of rand_logpdf is one b2b_chain_sample_vjp_f32 call with the
# forward's seed; the tangent of td is structural in its transform and its MvNormal.
function ChainRulesCore.rrule(::typeof(rand_logpdf), td::TransformedDistribution{<:MvNormal}, n::Integer;
                              seed::UInt64=rand(UInt64), offset::UInt64=UInt64(0), column_offset::Integer=0)
    y, lq = rand_logpdf(td, n; seed=seed, offset=offset, column_offset=column_offset)
    function rand_logpdf_pullback((ȳ, q̄))
        ȳd = ȳ isa ChainRulesCore.AbstractZero ? nothing : CuMatrix{Float32}(ȳ)
        q̄d = q̄ isa ChainRulesCore.AbstractZero ? nothing : CuVector{Float32}(q̄)
        flow, base = rand_vjp(td, n, ȳd, q̄d; seed=seed, offset=offset, column_offset=column_offset)
        t̄ = ChainRulesCore.Tangent{typeof(td)}(dist=base_tangent(td.dist, base),
                                               transform=transform_tangent(td.transform, flow, Ref(0)))
        return NoTangent(), t̄, NoTangent()
    end
    return (y, lq), rand_logpdf_pullback
end

# logpdf(td::MvTransformed, y::Matrix) (src/transformed_distribution.jl:165-169): inverse chain + base
# MvNormal + (optionally) the batch sum in ONE fused launch per fusable segment.
function Distributions.logpdf(td::TransformedDistribution{<:MvNormal}, y::CuMatrix{Float32})
    is_device(td.transform) || return invoke(Distributions.logpdf, Tuple{TransformedDistribution,AbstractMatrix}, td, y)
    ds = descs(td.transform, true)
    term, keep = base_desc(td.dist)
    push!(ds, term)
    GC.@preserve keep last(run_chain(ds, y; y=nothing))
end

# ---- multi-GPU (one process per GPU): one NCCL sum of the batch log-density (SURVEY §8(e)) ------------
mutable struct Comm; handle::Ptr{Cvoid}; end
function unique_id()
    uid = Vector{UInt8}(undef, 128)
    check(ccall((:b2b_comm_unique_id, libb2b), Cint, (Ptr{UInt8},), uid))
    uid
end
function Comm(nranks::Integer, rank::Integer, uid::Vector{UInt8})       # uid from unique_id() on rank 0
    h = Ref{Ptr{Cvoid}}()
    check(ccall((:b2b_comm_init_rank, libb2b), Cint, (Ptr{Ptr{Cvoid}}, Cint, Cint, Ptr{UInt8}), h, nranks, rank, uid))
    Comm(h[])
end
allreduce_sum!(c::Comm, v::CuVector{Float64}) =
    check(ccall((:b2b_allreduce_sum_f64, libb2b), Cint, (Ptr{Cvoid}, CuPtr{Float64}, Int32, Ptr{Cvoid}),
                c.handle, pointer(v), length(v), stream_handle()))
destroy!(c::Comm) = check(ccall((:b2b_comm_destroy, libb2b), Cint, (Ptr{Cvoid},), c.handle))

# One process per GPU: call once, before allocating pinned host batches (CPU affinity + memory policy next to the GPU).
function numa_bind(device::Integer=CUDA.deviceid())
    node, ncpu = Ref{Int32}(-1), Ref{Int32}(0)
    check(ccall((:b2b_numa_bind_to_device, libb2b), Cint, (Int32, Ptr{Int32}, Ptr{Int32}), device, node, ncpu))
    return node[], ncpu[]
end

end # module
