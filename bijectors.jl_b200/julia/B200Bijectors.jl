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
using Functors: fmap
using SparseArrays: findnz
using Statistics: mean, var

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
const PLANAR, RADIAL, RQS, COUPLING_AFFINE, BATCHNORM, PERMUTE, STACKED_EW, MVNORMAL_DIAG = Int32.(1:8)
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
desc(cl::Coupling, ::Bool) = error("Coupling: only AffineConditioner laws run on the device path (no CPU fallback)")

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
# a whole-column elementwise law is a one-block Stacked
const ElementwiseLaw = Union{Shift{<:Real},Scale{<:Real},LeakyReLU{<:Real},Logit{<:Real,<:Real},TruncatedBijector{<:Real,<:Real}}

# ---- chains: Base.ComposedFunction trees are flattened inner-most first ------------------------------
flatten(f::ComposedFunction) = (flatten(f.inner)..., flatten(f.outer)...)
flatten(f) = (f,)
descs(f, inv::Bool) = inv ? [desc(b, true) for b in reverse(flatten(f))] : [desc(b, false) for b in flatten(f)]

const DeviceLayer = Union{PlanarLayer{<:CuVector{Float32}},RadialLayer{<:CuVector{Float32}},
                          RationalQuadraticSpline{<:CuMatrix{Float32}},InvertibleBatchNorm{<:CuVector{Float32}},
                          Coupling{<:AffineConditioner},Permute,Stacked}
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

# rand(rng, td, n) (src/transformed_distribution.jl:212-224): the base samples are generated INSIDE the chain kernel
# (Philox4x32-10 + Box-Muller); `seed` plays the role of rng, `column_offset` continues one stream across column shards.
function device_rand(td::TransformedDistribution{<:MvNormal}, n::Integer; seed::UInt64=rand(UInt64), offset::UInt64=UInt64(0),
                     column_offset::Integer=0)
    ds = descs(td.transform, false)
    D = length(td.dist)
    μ, σ = cu(Float32.(mean(td.dist))), cu(Float32.(sqrt.(var(td.dist))))
    y = CuMatrix{Float32}(undef, D, n)
    ws_bytes = ccall((:b2b_chain_workspace_bytes, libb2b), Csize_t,
                     (Ptr{LayerDesc}, Int32, Int32, Int64, Cint, Cint), ds, length(ds), D, n, true, false)
    ws = CuVector{UInt8}(undef, ws_bytes)
    GC.@preserve ds μ σ ws check(ccall((:b2b_chain_sample_f32, libb2b), Cint,
        (Ptr{LayerDesc}, Int32, CuPtr{Float32}, CuPtr{Float32}, UInt64, UInt64, Int64, CuPtr{Float32}, CuPtr{Float32},
         Int32, Int64, Int64, CuPtr{Cvoid}, Csize_t, Ptr{Cvoid}),
        ds, length(ds), pointer(μ), pointer(σ), seed, offset, column_offset, pointer(y), NULLF,
        D, n, stride(y, 2), pointer(ws), ws_bytes, stream_handle()))
    return y
end

# logpdf(td::MvTransformed, y::Matrix) (src/transformed_distribution.jl:165-169): inverse chain + base
# MvNormal + (optionally) the batch sum in ONE fused launch per fusable segment.
function Distributions.logpdf(td::TransformedDistribution{<:MvNormal}, y::CuMatrix{Float32})
    is_device(td.transform) || return invoke(Distributions.logpdf, Tuple{TransformedDistribution,AbstractMatrix}, td, y)
    ds = descs(td.transform, true)
    μ, σ = cu(Float32.(mean(td.dist))), cu(Float32.(sqrt.(var(td.dist))))
    push!(ds, LayerDesc(MVNORMAL_DIAG, 0, 0, 0, 0, 0, 0f0, 0f0, pointer(μ), pointer(σ), NULLF, NULLF, NULLI, NULLI))
    GC.@preserve μ σ last(run_chain(ds, y; y=nothing))
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
