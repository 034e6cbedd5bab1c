# AGPBlackwell.jl -- the thin Julia shim a maintainer adds on the reference side so that AbstractGPs.jl's
# dense hot path runs on libagp.so (hand-written sm_90a CUDA behind the C ABI of include/agp.h).
#
# Julia is NOT available in the build image, so this file is shipped as source and has never been
# executed (INTEGRATION.md lists what a maintainer should check first); every `ccall` below is mirrored 1:1 by the ctypes binding
# abstractgps.jl_b200/_cabi.py, which IS exercised by the test-suite -- the ABI is what is tested.
#
# Seams used (SURVEY.md s1, s8b): ordinary multiple dispatch on
#   FiniteGP{<:GP{<:Union{ZeroMean,ConstMean,CustomMean},<:SupportedKernel}, <:Inputs, <:Diagonal}
# for logpdf / posterior / rand / elbo, and a device-resident factor type `DeviceCholesky` that slots
# into PosteriorGP.data.C with methods for the operator set of src/util/common_covmat_ops.jl.
# Anything else (other kernels, dense Sigma_y, ...) falls through to the stock reference methods.
module AGPBlackwell

using AbstractGPs, KernelFunctions, LinearAlgebra, FillArrays
import AbstractGPs: posterior, mean_and_var, elbo, approx_log_evidence, FiniteGP, PosteriorGP, VFE, DTC, GP
import AbstractGPs: Xt_invA_X, Xt_invA_Y, diag_Xt_invA_X, tr_Xt_invA_X
import Distributions: logpdf
import Random

const libagp = get(ENV, "AGP_LIB", "libagp.so")

# ---- POD structs of include/agp.h ------------------------------------------------------------
struct AgpKernelFactor; family::Int32; transform::Int32; scale::Float64; param::Float64; ard::Ptr{Cvoid}; r::Ptr{Cvoid}; end
struct AgpKernelComposite; nterms::Int32; nfactors::Ptr{Int32}; variance::Ptr{Float64}; factors::Ptr{AgpKernelFactor}; end
# `composite` (agp.h agp_kernel_composite) is read only for family AGP_COMPOSITE; single kernels pass C_NULL
struct AgpKernel; family::Int32; transform::Int32; variance::Float64; scale::Float64; linear_c::Float64; ard::Ptr{Cvoid}; composite::Ptr{AgpKernelComposite}; end
struct AgpMean;   kind::Int32; c::Float64; v::Ptr{Cvoid}; end
struct AgpNoise;  kind::Int32; s::Float64; v::Ptr{Cvoid}; end
const AGP_F32, AGP_F64 = Int32(0), Int32(1)
const AGP_POINT_MAJOR, AGP_FEATURE_MAJOR = Int32(0), Int32(1)
agp_dtype(::Type{Float32}) = AGP_F32
agp_dtype(::Type{Float64}) = AGP_F64

mutable struct Ctx
    h::Ptr{Cvoid}
    lock::ReentrantLock          # a ctx is not re-entrant (agp.h "Conventions")
end
const CTX = Ref{Union{Nothing,Ctx}}(nothing)
function ctx()
    if CTX[] === nothing
        h = Ref{Ptr{Cvoid}}(C_NULL)
        rc = ccall((:agp_init, libagp), Int32, (Ptr{Ptr{Cvoid}}, Int32, Ptr{Cvoid}), h, 0, C_NULL)
        rc == 0 || error("agp_init failed ($rc): no CUDA device? (there is no CPU fallback)")
        CTX[] = Ctx(h[], ReentrantLock())
    end
    return CTX[]
end

function check(c::Ctx, rc::Int32)
    rc == 0 && return
    msg = unsafe_string(ccall((:agp_last_error, libagp), Cstring, (Ptr{Cvoid},), c.h))
    rc == 1 && throw(PosDefException(ccall((:agp_last_info, libagp), Int64, (Ptr{Cvoid},), c.h)))  # cholesky(.) behaviour
    rc == 2 && throw(DimensionMismatch(msg))
    error("libagp status $rc: $msg")
end

# ---- kernel / mean / noise translation ----------------------------------------------------------
const Stationary = Union{SqExponentialKernel,Matern12Kernel,Matern32Kernel,Matern52Kernel}
family(::SqExponentialKernel) = Int32(0); family(::Matern12Kernel) = Int32(1)
family(::Matern32Kernel) = Int32(2);      family(::Matern52Kernel) = Int32(3); family(::LinearKernel) = Int32(4)

# Single kernels the engine implements: a base kernel wrapped in any nesting of ScaledKernel / TransformedKernel{Scale|ARD}.
# Sums, products and the factor-only families are claimed separately (`composite_supported`, exact path only); everything
# else is NOT claimed: the methods below `invoke` the stock reference method.
supported(::Union{Stationary,LinearKernel}) = true
supported(k::ScaledKernel) = supported(k.kernel)
supported(k::TransformedKernel{<:Any,<:Union{ScaleTransform,ARDTransform}}) = supported(k.kernel)
supported(::Kernel) = false
supported(::Union{AbstractGPs.ZeroMean,AbstractGPs.ConstMean,AbstractGPs.CustomMean}) = true
supported(::AbstractGPs.MeanFunction) = false
supported(f::GP) = supported(f.kernel) && supported(f.mean)
supported(::Any) = false

# flattened description: (family, sigma_f^2, linear c, per-dimension input scaling w) with w === nothing (identity),
# a scalar (ScaleTransform) or a vector (ARDTransform).  (k o t1) o t2 evaluates k(t1(t2(x))): diagonal scalings commute,
# so nested transforms multiply (the Python mirror's `_chain`).
flat(k::Union{Stationary,LinearKernel}) = (family(k), 1.0, k isa LinearKernel ? Float64(only(k.c)) : 0.0, nothing)
function flat(k::ScaledKernel)
    fam, var, c, w = flat(k.kernel)
    (fam, var * Float64(only(k.σ²)), c * 1.0, w)      # sigma^2 * (x'y + c) keeps c inside: the engine applies variance to both
end
combine(::Nothing, t) = t
combine(w, t) = w .* t
function flat(k::TransformedKernel{<:Any,<:ScaleTransform})
    fam, var, c, w = flat(k.kernel)
    (fam, var, c, combine(w, Float64(only(k.transform.s))))
end
function flat(k::TransformedKernel{<:Any,<:ARDTransform})
    fam, var, c, w = flat(k.kernel)
    (fam, var, c, combine(w, Float64.(k.transform.v)))
end
# returns (AgpKernel, keepalive)
function kernel_spec(k, T)
    fam, var, c, w = flat(k)
    w === nothing && return (AgpKernel(fam, 0, var, 1.0, c, C_NULL, C_NULL), nothing)
    w isa Real && return (AgpKernel(fam, 1, var, Float64(w), c, C_NULL, C_NULL), nothing)
    v = convert(Vector{T}, w)
    return (AgpKernel(fam, 2, var, 1.0, c, pointer(v), C_NULL), v)
end
# ---- composite kernels: KernelSum / KernelProduct / ScaledKernel / TransformedKernel trees (agp.h agp_kernel_composite) --
# The tree is flattened into a sum of product terms exactly as the Python mirror's `_walk` does: a sum concatenates its
# children's terms, a product distributes over them, a ScaledKernel's sigma^2 multiplies into every term below it and a
# TransformedKernel's scaling into every factor below it.  Within AGP_COMPOSITE_MAX terms and factors in all, the exact
# single-GPU methods claim the tree; anything else (and every VFE method) falls through to the stock reference methods.
const AGP_COMPOSITE = Int32(9)
const AGP_COMPOSITE_MAX = 8
const FactorOnly = Union{RationalQuadraticKernel,PeriodicKernel,WhiteKernel,ConstantKernel}
family(::RationalQuadraticKernel) = Int32(5); family(::PeriodicKernel) = Int32(6)
family(::WhiteKernel) = Int32(7);             family(::ConstantKernel) = Int32(8)

euclidean(k) = !hasproperty(k, :metric) || nameof(typeof(k.metric)) === :Euclidean
composite_ok(k::Union{Stationary,LinearKernel,FactorOnly}) = euclidean(k)
composite_ok(k::ScaledKernel) = composite_ok(k.kernel)
composite_ok(k::TransformedKernel{<:Any,<:Union{ScaleTransform,ARDTransform}}) = composite_ok(k.kernel)
composite_ok(k::Union{KernelSum,KernelProduct}) = all(composite_ok, k.kernels)
composite_ok(::Any) = false

# terms of a tree: [(scalings, factors)], scalings = [(ScaledKernel, path)], factors = [(leaf, path, transforms)],
# transforms = [(TransformedKernel, path)] innermost first.  A path is the list of child positions from the root (the
# `kernel` field of a ScaledKernel / TransformedKernel is child 1); the rrule addresses the tangent by it, so a parameter
# that flattening copies into several terms collects every copy's gradient.
walk(k::Union{Stationary,LinearKernel,FactorOnly}, p) = Any[(Any[], Any[(k, p, Any[])])]
walk(k::ScaledKernel, p) = Any[(vcat(Any[(k, p)], s), f) for (s, f) in walk(k.kernel, [p; 1])]
walk(k::TransformedKernel, p) = Any[(s, Any[(l, lp, vcat(tr, Any[(k, p)])) for (l, lp, tr) in f]) for (s, f) in walk(k.kernel, [p; 1])]
walk(k::KernelSum, p) = reduce(vcat, [walk(c, [p; i]) for (i, c) in enumerate(k.kernels)])
function walk(k::KernelProduct, p)
    terms = Any[(Any[], Any[])]
    for (i, c) in enumerate(k.kernels)
        ct = walk(c, [p; i])
        terms = Any[(vcat(a[1], b[1]), vcat(a[2], b[2])) for a in terms for b in ct]
    end
    return terms
end
walk(k) = walk(k, Int[])

within_limits(terms) = length(terms) <= AGP_COMPOSITE_MAX && sum(t -> length(t[2]), terms) <= AGP_COMPOSITE_MAX
composite_supported(k) = !supported(k) && composite_ok(k) && within_limits(walk(k))

# the exact single-GPU methods claim single kernels and composites; the VFE methods keep `supported` (single kernels)
claimed(f::GP) = (supported(f.kernel) || composite_supported(f.kernel)) && supported(f.mean)
claimed(::Any) = false

sigma2(s::ScaledKernel) = Float64(only(s.σ²))
tscale(t::TransformedKernel) = t.transform isa ScaleTransform ? Float64(only(t.transform.s)) : Float64.(t.transform.v)
prod_except(xs, j, D) = foldl((a, b) -> a .* b, (xs[i] for i in eachindex(xs) if i != j); init=D === nothing ? 1.0 : ones(D))

# (AGP_T_*, s, v) of a factor: its transform chain multiplied out
function transform_of(tr, D)
    isempty(tr) && return (Int32(0), 1.0, nothing)
    ws = [tscale(t) for (t, _) in tr]
    all(w -> w isa Real, ws) && return (Int32(1), prod(ws), nothing)
    v = prod_except(ws, 0, D)
    length(v) == D || throw(DimensionMismatch("ARD weights have length $(length(v)), inputs have D = $D"))
    return (Int32(2), 1.0, v)
end
factor_param(k::RationalQuadraticKernel) = Float64(only(k.α))
factor_param(k::Union{LinearKernel,ConstantKernel}) = Float64(only(k.c))
factor_param(::Any) = 0.0
function periodic_r(k::PeriodicKernel, D)
    length(k.r) in (1, D) || throw(DimensionMismatch("PeriodicKernel r has length $(length(k.r)), inputs have D = $D"))
    return length(k.r) == 1 ? fill(Float64(only(k.r)), D) : Float64.(k.r)
end

# returns (AgpKernel, keepalive) for a composite tree
function composite_spec(k, T, D)
    terms = walk(k)
    keep = Any[]
    nf = Int32[length(f) for (_, f) in terms]
    var = Float64[prod(sigma2(s) for (s, _) in sc; init=1.0) for (sc, _) in terms]
    facs = AgpKernelFactor[]
    for (_, fs) in terms, (leaf, _, tr) in fs
        kind, s, v = transform_of(tr, D)
        ard = C_NULL
        if v !== nothing
            va = convert(Vector{T}, v); push!(keep, va); ard = pointer(va)
        end
        r = C_NULL
        if leaf isa PeriodicKernel
            ra = convert(Vector{T}, periodic_r(leaf, D)); push!(keep, ra); r = pointer(ra)
        end
        push!(facs, AgpKernelFactor(family(leaf), kind, s, factor_param(leaf), ard, r))
    end
    comp = [AgpKernelComposite(Int32(length(terms)), pointer(nf), pointer(var), pointer(facs))]
    push!(keep, nf, var, facs, comp)
    return (AgpKernel(AGP_COMPOSITE, 0, 1.0, 1.0, 0.0, C_NULL, pointer(comp)), keep)
end
kernel_spec(k, T, D) = supported(k) ? kernel_spec(k, T) : composite_spec(k, T, D)

mean_spec(::AbstractGPs.ZeroMean, x, T) = (AgpMean(0, 0.0, C_NULL), nothing)
mean_spec(m::AbstractGPs.ConstMean, x, T) = (AgpMean(1, Float64(m.c), C_NULL), nothing)
function mean_spec(m::AbstractGPs.CustomMean, x, T)      # arbitrary closure: evaluated host-side
    v = convert(Vector{T}, AbstractGPs.mean_vector(m, x)); (AgpMean(2, 0.0, pointer(v)), v)
end
noise_spec(Σ::Diagonal{<:Any,<:Fill}, T) = (AgpNoise(0, Float64(Σ.diag.value), C_NULL), nothing)
function noise_spec(Σ::Diagonal, T); v = convert(Vector{T}, Σ.diag); (AgpNoise(1, 0.0, pointer(v)), v); end

points(x::ColVecs{T}) where {T} = (x.X, AGP_POINT_MAJOR, size(x.X, 1))
points(x::RowVecs{T}) where {T} = (x.X, AGP_FEATURE_MAJOR, size(x.X, 2))
points(x::AbstractVector{T}) where {T<:Real} = (x, AGP_POINT_MAJOR, 1)
# a second input collection (inducing / test points) in the SAME storage order as the first: the ABI takes one layout flag
same_layout(z::ColVecs, layout) = layout == AGP_POINT_MAJOR ? z.X : permutedims(z.X)
same_layout(z::RowVecs, layout) = layout == AGP_FEATURE_MAJOR ? z.X : permutedims(z.X)
same_layout(z::AbstractVector{<:Real}, layout) = z

# ---- device factor (boundary #2) --------------------------------------------------------------
mutable struct DeviceCholesky{T}
    h::Ptr{Cvoid}
    n::Int
    function DeviceCholesky{T}(h, n) where {T}
        C = new{T}(h, n)
        finalizer(c -> ccall((:agp_post_free, libagp), Int32, (Ptr{Cvoid},), c.h), C)
    end
end
function Base.getproperty(C::DeviceCholesky{T}, s::Symbol) where {T}
    s === :U || return getfield(C, s)
    U = Matrix{T}(undef, C.n, C.n)
    check(ctx(), ccall((:agp_post_factor_export, libagp), Int32, (Ptr{Cvoid}, Ptr{Cvoid}), C.h, U))
    return UpperTriangular(U)
end
function solve_lower(C::DeviceCholesky{T}, B::AbstractVecOrMat) where {T}      # C.U' \ B
    Bm = convert(Matrix{T}, reshape(B, C.n, :)); V = similar(Bm)
    check(ctx(), ccall((:agp_post_solve_lower, libagp), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ptr{Cvoid}), C.h, Bm, size(Bm, 2), V))
    return B isa AbstractVector ? vec(V) : V
end
Xt_invA_X(A::DeviceCholesky, x::AbstractVector) = sum(abs2, solve_lower(A, x))
Xt_invA_X(A::DeviceCholesky, X::AbstractMatrix) = (V = solve_lower(A, X); Symmetric(V'V))
Xt_invA_Y(X::AbstractVecOrMat, A::DeviceCholesky, Y::AbstractVecOrMat) = solve_lower(A, X)' * solve_lower(A, Y)
diag_Xt_invA_X(A::DeviceCholesky, X::AbstractVecOrMat) = AbstractGPs.diag_At_A(solve_lower(A, X))
tr_Xt_invA_X(A::DeviceCholesky, X::AbstractVecOrMat) = sum(abs2, solve_lower(A, X))

# ---- fused fit: logpdf + posterior from ONE Gram and ONE factorisation ---------------------------
const DevInputs{T} = Union{Vector{T},ColVecs{T},RowVecs{T}}
const DevFiniteGP{T} = FiniteGP{<:GP,<:DevInputs{T},<:Diagonal}

function fit(fx::DevFiniteGP{T}, Y::AbstractVecOrMat; want_post::Bool=true) where {T<:Union{Float32,Float64}}
    c = ctx()
    X, layout, D = points(fx.x)
    Ym = convert(Matrix{T}, reshape(Y, length(fx), :))
    ks, k1 = kernel_spec(fx.f.kernel, T, D); ms, k2 = mean_spec(fx.f.mean, fx.x, T); ns, k3 = noise_spec(fx.Σy, T)
    lp = Vector{T}(undef, size(Ym, 2)); α = Vector{T}(undef, length(fx)); post = Ref{Ptr{Cvoid}}(C_NULL)
    lock(c.lock) do
        GC.@preserve X Ym k1 k2 k3 begin
            check(c, ccall((:agp_fit, libagp), Int32,
                (Ptr{Cvoid}, Int32, Ref{AgpKernel}, Ref{AgpMean}, Ref{AgpNoise}, Int32, Ptr{Cvoid}, Int64, Int32,
                 Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}),
                c.h, agp_dtype(T), ks, ms, ns, layout, X, length(fx), D, Ym, size(Ym, 2), lp,
                want_post ? pointer(α) : C_NULL, want_post ? post : C_NULL))
        end
    end
    lpv = Y isa AbstractVector ? lp[1] : lp
    want_post || return lpv, nothing
    δ = Ym[:, 1] - AbstractGPs.mean(fx)
    return lpv, PosteriorGP(fx.f, (α=α, C=DeviceCholesky{T}(post[], length(fx)), x=fx.x, δ=δ))
end

# replaces src/finite_gp_projection.jl:306-311 and src/exact_gpr_posterior.jl:29-35 for the device types
# priors the engine does not implement fall through to the reference's own methods (Julia dispatch, not a CPU fallback
# inside the engine)
logpdf(fx::DevFiniteGP{T}, Y::AbstractVecOrMat{<:Real}) where {T} =
    claimed(fx.f) ? fit(fx, Y; want_post=false)[1] : invoke(logpdf, Tuple{FiniteGP,typeof(Y)}, fx, Y)
posterior(fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T} =
    claimed(fx.f) ? fit(fx, y)[2] : invoke(posterior, Tuple{FiniteGP,AbstractVector{<:Real}}, fx, y)

# replaces src/exact_gpr_posterior.jl:85-90 (+ src/finite_gp_projection.jl:154-158) with the fused cross-Gram path
const DevPosterior = PosteriorGP{<:GP,<:NamedTuple{(:α, :C, :x, :δ),<:Tuple{Any,DeviceCholesky,Any,Any}}}
mean_and_var(fx::FiniteGP{<:DevPosterior,<:DevInputs{T},<:Diagonal}) where {T} = post_mean_var_primal(fx, false)
# zero_mean: the means of the zero-mean prior at x* (the CustomMean split of the mean_and_var rule below)
function post_mean_var_primal(fx::FiniteGP{<:DevPosterior,<:DevInputs{T},<:Diagonal}, zero_mean::Bool) where {T}
    p = fx.f; c = ctx(); Xs, layout, D = points(fx.x); M = length(fx)
    ms, k2 = zero_mean ? mean_spec(AbstractGPs.ZeroMean(), fx.x, T) : mean_spec(p.prior.mean, fx.x, T)
    ns, k3 = noise_spec(fx.Σy, T)
    μ = Vector{T}(undef, M); v = Vector{T}(undef, M)
    lock(c.lock) do
        GC.@preserve Xs k2 k3 check(c, ccall((:agp_post_mean_var, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ref{AgpMean}, Ref{AgpNoise}, Ptr{Cvoid}, Ptr{Cvoid}),
            p.data.C.h, layout, Xs, M, ms, ns, μ, v))
    end
    return μ, v
end

# FiniteGP over a device posterior: logpdf / rand / sequential conditioning stay on the device
# (src/finite_gp_projection.jl:306-318, :233-237 and src/exact_gpr_posterior.jl:46-56 for f = PosteriorGP)
const DevPostFiniteGP{T} = FiniteGP{<:DevPosterior,<:DevInputs{T},<:Diagonal}
function logpdf(fx::DevPostFiniteGP{T}, Y::AbstractVecOrMat{<:Real}) where {T}
    p = fx.f; c = ctx(); Xs, layout, D = points(fx.x); M = length(fx)
    Ym = convert(Matrix{T}, reshape(Y, M, :)); lp = Vector{T}(undef, size(Ym, 2))
    ms, k2 = mean_spec(p.prior.mean, fx.x, T); ns, k3 = noise_spec(fx.Σy, T)
    lock(c.lock) do
        GC.@preserve Xs Ym k2 k3 check(c, ccall((:agp_post_logpdf, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ref{AgpMean}, Ref{AgpNoise}, Ptr{Cvoid}, Int32, Ptr{Cvoid}),
            p.data.C.h, layout, Xs, M, ms, ns, Ym, size(Ym, 2), lp))
    end
    return Y isa AbstractVector ? lp[1] : lp
end
Random.rand(rng::Random.AbstractRNG, fx::DevPostFiniteGP{T}, S::Int) where {T} = post_rand_primal(rng, fx, S, false)[1]
function posterior(fx::DevPostFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    p = fx.f; c = ctx(); X2, layout, D = points(fx.x); N2 = length(fx); N1 = p.data.C.n
    yv = convert(Vector{T}, y); α = Vector{T}(undef, N1 + N2); post = Ref{Ptr{Cvoid}}(C_NULL)
    ms, k2 = mean_spec(p.prior.mean, fx.x, T); ns, k3 = noise_spec(fx.Σy, T)
    lock(c.lock) do
        GC.@preserve X2 yv k2 k3 check(c, ccall((:agp_post_extend, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ref{AgpMean}, Ref{AgpNoise}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}),
            p.data.C.h, layout, X2, N2, yv, ms, ns, α, post))
    end
    δ = vcat(p.data.δ, yv - AbstractGPs.mean_vector(p.prior.mean, fx.x))
    return PosteriorGP(p.prior, (α=α, C=DeviceCholesky{T}(post[], N1 + N2), x=vcat(p.data.x, fx.x), δ=δ))
end

# replaces rand(rng, fx, S) src/finite_gp_projection.jl:233-237: the normals come from the caller's rng
function Random.rand(rng::Random.AbstractRNG, fx::DevFiniteGP{T}, S::Int) where {T}
    claimed(fx.f) || return invoke(Random.rand, Tuple{Random.AbstractRNG,FiniteGP,Int}, rng, fx, S)
    c = ctx(); X, layout, D = points(fx.x); Z = randn(rng, T, length(fx), S); out = similar(Z)
    ks, k1 = kernel_spec(fx.f.kernel, T, D); ms, k2 = mean_spec(fx.f.mean, fx.x, T); ns, k3 = noise_spec(fx.Σy, T)
    lock(c.lock) do
        GC.@preserve X k1 k2 k3 check(c, ccall((:agp_rand, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ref{AgpKernel}, Ref{AgpMean}, Ref{AgpNoise}, Int32, Ptr{Cvoid}, Int64, Int32, Ptr{Cvoid}, Int32, Ptr{Cvoid}),
            c.h, agp_dtype(T), ks, ms, ns, layout, X, length(fx), D, Z, S, out))
    end
    return out
end

# replaces approx_log_evidence(::VFE / ::DTC, fx, y) src/sparse_approximations.jl:248-254, :282-286: ONE streamed pass
# returns both objectives (elbo, dtc)
function sparse_objectives(fz::FiniteGP, fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    fz.f === fx.f || throw(ArgumentError("the inducing and the data FiniteGP must share the prior"))
    length(y) == length(fx) || throw(DimensionMismatch("length(fx) = $(length(fx)) but length(y) = $(length(y))"))
    c = ctx(); X, layout, D = points(fx.x); Z = same_layout(fz.x, layout)
    ks, k1 = kernel_spec(fx.f.kernel, T); ms, k2 = mean_spec(fx.f.mean, fx.x, T)
    ns, k3 = noise_spec(fx.Σy, T); js, k4 = noise_spec(fz.Σy, T)
    yv = convert(Vector{T}, y); out = Vector{T}(undef, 2)
    lock(c.lock) do
        GC.@preserve X Z yv out k1 k2 k3 k4 check(c, ccall((:agp_vfe_elbo, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ref{AgpKernel}, Ref{AgpMean}, Ref{AgpNoise}, Int32, Ptr{Cvoid}, Int64, Int32, Ptr{Cvoid}, Int64,
             Ref{AgpNoise}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
            c.h, agp_dtype(T), ks, ms, ns, layout, X, length(fx), D, Z, length(fz), js, yv, pointer(out, 1), pointer(out, 2)))
    end
    return out[1], out[2]
end
approx_log_evidence(vfe::VFE, fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T} =
    supported(fx.f) ? sparse_objectives(vfe.fz, fx, y)[1] : invoke(approx_log_evidence, Tuple{VFE,FiniteGP,AbstractVector{<:Real}}, vfe, fx, y)
approx_log_evidence(dtc::DTC, fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T} =
    supported(fx.f) ? sparse_objectives(dtc.fz, fx, y)[2] : invoke(approx_log_evidence, Tuple{DTC,FiniteGP,AbstractVector{<:Real}}, dtc, fx, y)

# ---- posterior(::VFE, fx, y) src/sparse_approximations.jl:58-75 and its predictive mean_and_var :212-217 ------------
# The reference's ApproxPosteriorGP caches host matrices; the device posterior keeps chol(K_zz), chol(A A' + I) and
# m_eps in HBM behind an agp_vfe_post handle.
mutable struct DeviceApproxPosterior{T,Tprior,Tz} <: AbstractGPs.AbstractGP
    h::Ptr{Cvoid}
    prior::Tprior
    z::Tz
    function DeviceApproxPosterior{T}(h, prior, z) where {T}
        p = new{T,typeof(prior),typeof(z)}(h, prior, z)
        finalizer(q -> ccall((:agp_vfe_post_free, libagp), Int32, (Ptr{Cvoid},), q.h), p)
    end
end
function posterior(vfe::Union{VFE,DTC}, fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    supported(fx.f) || return invoke(posterior, Tuple{typeof(vfe),FiniteGP,AbstractVector{<:Real}}, vfe, fx, y)
    fz = vfe.fz
    fz.f === fx.f || throw(ArgumentError("the inducing and the data FiniteGP must share the prior"))
    c = ctx(); X, layout, D = points(fx.x); Z = same_layout(fz.x, layout)
    ks, k1 = kernel_spec(fx.f.kernel, T); ms, k2 = mean_spec(fx.f.mean, fx.x, T)
    ns, k3 = noise_spec(fx.Σy, T); js, k4 = noise_spec(fz.Σy, T)
    yv = convert(Vector{T}, y); post = Ref{Ptr{Cvoid}}(C_NULL)
    lock(c.lock) do
        GC.@preserve X Z yv k1 k2 k3 k4 check(c, ccall((:agp_vfe_fit, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ref{AgpKernel}, Ref{AgpMean}, Ref{AgpNoise}, Int32, Ptr{Cvoid}, Int64, Int32, Ptr{Cvoid}, Int64,
             Ref{AgpNoise}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}),
            c.h, agp_dtype(T), ks, ms, ns, layout, X, length(fx), D, Z, length(fz), js, yv, post))
    end
    return DeviceApproxPosterior{T}(post[], fx.f, fz.x)
end
function mean_and_var(fx::FiniteGP{<:DeviceApproxPosterior{T},<:DevInputs{T},<:Diagonal}) where {T}
    p = fx.f; c = ctx(); Xs, layout, D = points(fx.x); M = length(fx)
    μ = Vector{T}(undef, M); v = Vector{T}(undef, M)
    lock(c.lock) do
        GC.@preserve Xs check(c, ccall((:agp_vfe_mean_var, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ptr{Cvoid}), p.h, layout, Xs, M, μ, v))
    end
    # the handle applies Zero / Const prior means; a closure mean is evaluated host-side (src/mean_function.jl:52-55)
    p.prior.mean isa AbstractGPs.CustomMean && (μ .+= AbstractGPs.mean_vector(p.prior.mean, fx.x))
    return μ, v .+ diag(fx.Σy)
end
AbstractGPs.mean_and_var(p::DeviceApproxPosterior{T}, x::DevInputs{T}) where {T} = mean_and_var(p(x, zero(T)))
AbstractGPs.mean(fx::FiniteGP{<:DeviceApproxPosterior}) = mean_and_var(fx)[1]
AbstractGPs.var(fx::FiniteGP{<:DeviceApproxPosterior}) = mean_and_var(fx)[2]

# ---- reverse-mode rule for logpdf (test/finite_gp_projection.jl:152-178, examples/1-mauna-loa/script.jl:200-242) ------
# agp_post_logpdf_grad returns, from the factor of ONE fit, d logpdf / d (total sigma_f^2, total ScaleTransform factor,
# LinearKernel c, scalar noise, constant mean, total ARD weights) and the per-point noise gradient.  `logpdf_and_gradient`
# exposes them flat; the `rrule` maps them back onto the nested kernel structs (chain rule through the products the shim
# forms in `flat`: sigma_f^2 = prod of the ScaledKernel factors, w = prod of the transform scalings).  The rrules take the
# same gradients and, from the same C^-1, the gradient with respect to the inputs x through one agp_post_logpdf_grad_x call
# (`logpdf_gradients`), so a network that computes x (examples/2-deep-kernel-learning) trains through the GP term.  A
# CustomMean closure is not differentiated (with respect to its parameters or to x).
import ChainRulesCore
const CRC = ChainRulesCore

function logpdf_and_gradient(fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    lp, post = fit(fx, y)
    D = points(fx.x)[3]; N = length(fx)
    g = Vector{Float64}(undef, 5 + D); nd = Vector{T}(undef, N)
    c = ctx()
    lock(c.lock) do
        GC.@preserve g nd check(c, ccall((:agp_post_logpdf_grad, libagp), Int32, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Cvoid}), post.data.C.h, g, nd))
    end
    return lp, (variance=g[1], scale=g[2], linear_c=g[3], noise=g[4], mean_c=g[5], ard=g[6:end], noise_diag=nd, y=-post.data.α)
end

# the rrules' single call: (lp, post, g, noise_diag, x gradient shaped like fx.x's storage) from one fit and ONE
# agp_post_logpdf_grad_x (C^-1 is formed once for the hyper-parameters and the inputs); glen = length of g
function logpdf_gradients(fx::DevFiniteGP{T}, y::AbstractVector{<:Real}, glen) where {T}
    lp, post = fit(fx, y)
    X, layout, D = points(fx.x); N = length(fx)
    g = Vector{Float64}(undef, glen(post, D)); nd = Vector{T}(undef, N); xg = similar(X, T)
    c = ctx()
    lock(c.lock) do
        GC.@preserve g nd xg check(c, ccall((:agp_post_logpdf_grad_x, libagp), Int32,
            (Ptr{Cvoid}, Ptr{Float64}, Ptr{Cvoid}, Int32, Ptr{Cvoid}), post.data.C.h, g, nd, layout, xg))
    end
    return lp, post, g, nd, xg
end

# tangent of the inputs: the container's own field for ColVecs / RowVecs, a plain vector otherwise
x_tangent(x::ColVecs, xg) = CRC.Tangent{typeof(x)}(; X=xg)
x_tangent(x::RowVecs, xg) = CRC.Tangent{typeof(x)}(; X=xg)
x_tangent(x::AbstractVector{<:Real}, xg) = xg

# tangent of a (nested) kernel: `tot` carries the flattened totals the gradients refer to
kernel_tangent(k::Stationary, g, var, w) = CRC.NoTangent()
kernel_tangent(k::LinearKernel, g, var, w) = CRC.Tangent{typeof(k)}(; c=[g.linear_c])
function kernel_tangent(k::ScaledKernel, g, var, w)          # d/d sigma_i^2 = d/d var * var / sigma_i^2
    CRC.Tangent{typeof(k)}(; kernel=kernel_tangent(k.kernel, g, var, w), σ²=[g.variance * var / only(k.σ²)])
end
function kernel_tangent(k::TransformedKernel{<:Any,<:ScaleTransform}, g, var, w)
    s_i = only(k.transform.s)
    ds = w isa Real ? g.scale * w / s_i : sum(g.ard .* w) / s_i      # scalar layer under vector totals: sum over dimensions
    CRC.Tangent{typeof(k)}(; kernel=kernel_tangent(k.kernel, g, var, w), transform=CRC.Tangent{typeof(k.transform)}(; s=[ds]))
end
function kernel_tangent(k::TransformedKernel{<:Any,<:ARDTransform}, g, var, w)
    dv = g.ard .* w ./ k.transform.v                                    # d/d v_i[d] = d/d w[d] * w[d] / v_i[d]
    CRC.Tangent{typeof(k)}(; kernel=kernel_tangent(k.kernel, g, var, w), transform=CRC.Tangent{typeof(k.transform)}(; v=dv))
end
mean_tangent(m::AbstractGPs.ConstMean, g) = CRC.Tangent{typeof(m)}(; c=g.mean_c)
mean_tangent(m, g) = CRC.NoTangent()
noise_tangent(Σ::Diagonal{<:Any,<:Fill}, g) = CRC.Tangent{typeof(Σ)}(; diag=CRC.Tangent{typeof(Σ.diag)}(; value=g.noise))
noise_tangent(Σ::Diagonal, g) = CRC.Tangent{typeof(Σ)}(; diag=collect(g.noise_diag))

# ---- composite kernels: the descriptor gradient (agp.h, agp_post_logpdf_grad) mapped onto the tree by the chain rule ----
# Slots from g[6] (1-based): per term d/d v_t, then per factor d/d s or d/d v[1:D], d/d param, d/d r[1:D].  v_t is the
# product of the term's ScaledKernel sigma^2, a factor's s / v the product of its transforms: each node receives the slot's
# gradient times the product of the OTHER nodes (no division by a parameter), summed over every copy flattening made.
function composite_grads(k, D, g)
    acc = Dict{Vector{Int},Any}()
    add!(p, x) = (acc[p] = haskey(acc, p) ? acc[p] .+ x : x)
    pos = 6
    for (sc, fs) in walk(k)
        σ = [sigma2(s) for (s, _) in sc]
        for (j, (_, p)) in enumerate(sc)
            add!(p, g[pos] * prod_except(σ, j, nothing))
        end
        pos += 1
        for (leaf, lp, tr) in fs
            kind, _, _ = transform_of(tr, D)
            ws = [tscale(t) for (t, _) in tr]
            if kind == 1
                for (j, (_, p)) in enumerate(tr)
                    add!(p, g[pos] * prod_except(ws, j, nothing))
                end
                pos += 1
            elseif kind == 2
                gv = g[pos:pos+D-1]
                for (j, (t, p)) in enumerate(tr)
                    c = gv .* prod_except(ws, j, D)
                    add!(p, t.transform isa ScaleTransform ? sum(c) : c)
                end
                pos += D
            end
            if leaf isa Union{RationalQuadraticKernel,LinearKernel,ConstantKernel}
                add!(lp, g[pos]); pos += 1
            end
            if leaf isa PeriodicKernel
                gr = g[pos:pos+D-1]
                add!(lp, length(leaf.r) == 1 ? [sum(gr)] : gr); pos += D
            end
        end
    end
    return acc
end

# tangent of the tree from the per-path gradients (scaled by the cotangent d)
ctangent(k::Union{Stationary,WhiteKernel}, p, acc, d) = CRC.NoTangent()
ctangent(k::LinearKernel, p, acc, d) = CRC.Tangent{typeof(k)}(; c=[d * get(acc, p, 0.0)])
ctangent(k::ConstantKernel, p, acc, d) = CRC.Tangent{typeof(k)}(; c=[d * get(acc, p, 0.0)])
ctangent(k::RationalQuadraticKernel, p, acc, d) = CRC.Tangent{typeof(k)}(; α=[d * get(acc, p, 0.0)])
ctangent(k::PeriodicKernel, p, acc, d) = CRC.Tangent{typeof(k)}(; r=d .* get(acc, p, zeros(length(k.r))))
ctangent(k::ScaledKernel, p, acc, d) =
    CRC.Tangent{typeof(k)}(; kernel=ctangent(k.kernel, [p; 1], acc, d), σ²=[d * get(acc, p, 0.0)])
ctangent(k::TransformedKernel{<:Any,<:ScaleTransform}, p, acc, d) = CRC.Tangent{typeof(k)}(;
    kernel=ctangent(k.kernel, [p; 1], acc, d), transform=CRC.Tangent{typeof(k.transform)}(; s=[d * get(acc, p, 0.0)]))
ctangent(k::TransformedKernel{<:Any,<:ARDTransform}, p, acc, d) = CRC.Tangent{typeof(k)}(;
    kernel=ctangent(k.kernel, [p; 1], acc, d),
    transform=CRC.Tangent{typeof(k.transform)}(; v=d .* get(acc, p, zeros(length(k.transform.v)))))
function ctangent(k::Union{KernelSum,KernelProduct}, p, acc, d)
    ts = [ctangent(c, [p; i], acc, d) for (i, c) in enumerate(k.kernels)]
    CRC.Tangent{typeof(k)}(; kernels=k.kernels isa Tuple ? CRC.Tangent{typeof(k.kernels)}(ts...) : ts)
end

function composite_rrule(fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    D = points(fx.x)[3]
    lp, post, g, nd, xg = logpdf_gradients(fx, y, (post, D) -> ccall((:agp_post_grad_len, libagp), Int64, (Ptr{Cvoid},), post.data.C.h))
    acc = composite_grads(fx.f.kernel, D, g)
    function composite_pullback(Δ)
        d = CRC.unthunk(Δ)
        gs = (noise=d * g[4], mean_c=d * g[5], noise_diag=d .* nd)
        f̄ = CRC.Tangent{typeof(fx.f)}(; mean=mean_tangent(fx.f.mean, gs), kernel=ctangent(fx.f.kernel, Int[], acc, d))
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, d .* xg), Σy=noise_tangent(fx.Σy, gs))
        return CRC.NoTangent(), f̄x, -d .* post.data.α
    end
    return lp, composite_pullback
end

function CRC.rrule(::typeof(logpdf), fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    claimed(fx.f) && !supported(fx.f) && return composite_rrule(fx, y)
    supported(fx.f) || return nothing                                     # no rule: AD differentiates the stock method
    lp, post, gv, nd, xg = logpdf_gradients(fx, y, (post, D) -> 5 + D)
    g = (variance=gv[1], scale=gv[2], linear_c=gv[3], noise=gv[4], mean_c=gv[5], ard=gv[6:end], noise_diag=nd, y=-post.data.α)
    _, var, _, w = flat(fx.f.kernel)
    w === nothing && (w = 1.0)
    function logpdf_pullback(Δ)
        d = CRC.unthunk(Δ)
        gs = map(v -> v isa Number ? d * v : d .* v, g)
        f̄ = CRC.Tangent{typeof(fx.f)}(; mean=mean_tangent(fx.f.mean, gs), kernel=kernel_tangent(fx.f.kernel, gs, var, w))
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, d .* xg), Σy=noise_tangent(fx.Σy, gs))
        return CRC.NoTangent(), f̄x, gs.y
    end
    return lp, logpdf_pullback
end

# ---- reverse-mode rule for logpdf(fx, Y) with a matrix Y (test/finite_gp_projection.jl:165-178) ------------------------
# The forward pass is one fit that keeps the handle; the pullback receives the S-vector of cotangents Δ and makes ONE
# agp_post_logpdf_grad_cols call with lp_bar = Δ, so one factorisation and one C^-1 serve every column.
# loglikelihood(fx, Y) = sum(logpdf(fx, Y)) differentiates through this rule.  The tangents are mapped back by the helpers
# of the rules above; Ȳ is the tangent of Y.  A CustomMean's values go to the call again (the handle keeps none), and the
# closure is not differentiated, as in the vector rule.
function CRC.rrule(::typeof(logpdf), fx::DevFiniteGP{T}, Y::AbstractMatrix{<:Real}) where {T}
    claimed(fx.f) || return nothing                                       # no rule: AD differentiates the stock method
    lp, post = fit(fx, Y)
    c = ctx(); X, layout, D = points(fx.x); N = length(fx); S = size(Y, 2)
    Ym = convert(Matrix{T}, Y)
    ms, k2 = mean_spec(fx.f.mean, fx.x, T)
    composite = !supported(fx.f)
    function logpdf_matrix_pullback(Δ)
        Δ = CRC.unthunk(Δ)
        Δ isa CRC.AbstractZero && return CRC.NoTangent(), CRC.ZeroTangent(), CRC.ZeroTangent()
        w = convert(Vector{Float64}, Δ)
        glen = composite ? ccall((:agp_post_grad_len, libagp), Int64, (Ptr{Cvoid},), post.data.C.h) : 5 + D
        g = Vector{Float64}(undef, glen); nd = Vector{T}(undef, N); xg = similar(X, T); Ȳ = Matrix{T}(undef, N, S)
        lock(c.lock) do
            GC.@preserve Ym w g nd xg Ȳ k2 check(c, ccall((:agp_post_logpdf_grad_cols, libagp), Int32,
                (Ptr{Cvoid}, Ref{AgpMean}, Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Cvoid}, Ptr{Cvoid}, Int32,
                 Ptr{Cvoid}, Ptr{Cvoid}),
                post.data.C.h, ms, Ym, S, w, g, nd, C_NULL, layout, xg, Ȳ))
        end
        gs = (variance=g[1], scale=g[2], linear_c=g[3], noise=g[4], mean_c=g[5], ard=g[6:end], noise_diag=nd)
        if composite
            kt = ctangent(fx.f.kernel, Int[], composite_grads(fx.f.kernel, D, g), 1.0)
        else
            _, var, _, wt = flat(fx.f.kernel)
            kt = kernel_tangent(fx.f.kernel, gs, var, wt === nothing ? 1.0 : wt)
        end
        f̄ = CRC.Tangent{typeof(fx.f)}(; mean=mean_tangent(fx.f.mean, gs), kernel=kt)
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, xg), Σy=noise_tangent(fx.Σy, gs))
        return CRC.NoTangent(), f̄x, Ȳ
    end
    return lp, logpdf_matrix_pullback
end

# ---- reverse-mode rules for the held-out log-likelihood logpdf(posterior(fx, y)(x*, Σ*), y*) ----------------------------
# (examples/0-intro-1d/script.jl scores its models with it; validation-likelihood training maximises it.)
# posterior(fx, y) keeps the handle: its rule runs the primal and its pullback only re-routes a tangent of the DevPosterior
# -- prior -> fx.f, data.x -> fx.x, data.δ -> y and, since δ = y - m(x), minus its sum to a ConstMean, and data.C -> fx.Σy.
# logpdf over a DevPosterior makes ONE agp_post_pred_logpdf_grad call with lp_bar = Δ and returns the total derivatives
# in that tangent shape: the kernel through every block (K_xx, K_xs, K_ss), data.x, data.δ = ȳ, the prior mean through
# the test side only (the training side reaches it through data.δ), and in data.C the diagonal of the cotangent of
# C = K_xx + Σy as (noise = its trace, noise_diag = its diagonal): the part of C's cotangent that Σy receives (the kernel
# part is already in prior.kernel).  Every Tangent names only fields its primal has (FiniteGP: f, x, Σy; GP: mean, kernel;
# PosteriorGP: prior, data; data: α, C, x, δ).  fx.x, fx.Σy and Y get theirs directly.  A CustomMean closure is not
# differentiated, as in the rules above.
notangent(t) = t === nothing || t isa CRC.AbstractZero
# the c of a ConstMean's tangent as the AD system hands it back (a Tangent or a NamedTuple); 0 for no tangent
tangent_c(Δm) = notangent(Δm) ? 0.0 : Δm.c

function CRC.rrule(::typeof(posterior), fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    claimed(fx.f) || return nothing                                       # no rule: AD differentiates the stock method
    post = posterior(fx, y)
    function posterior_pullback(Δ)
        Δp = CRC.unthunk(Δ)
        notangent(Δp) && return CRC.NoTangent(), CRC.ZeroTangent(), CRC.ZeroTangent()
        Δd, Δf = Δp.data, Δp.prior
        ȳ = notangent(Δd) || notangent(Δd.δ) ? zeros(T, length(y)) : Δd.δ
        # a new ConstMean tangent from the scalar c's, rather than a sum of tangents of different wrappers
        m̄ = fx.f.mean isa AbstractGPs.ConstMean ?
            mean_tangent(fx.f.mean, (mean_c=(notangent(Δf) ? 0.0 : tangent_c(Δf.mean)) - sum(ȳ),)) : CRC.NoTangent()
        f̄ = CRC.Tangent{typeof(fx.f)}(; mean=m̄, kernel=notangent(Δf) ? CRC.NoTangent() : Δf.kernel)
        x̄ = notangent(Δd) || notangent(Δd.x) ? CRC.NoTangent() : Δd.x
        Σ̄ = notangent(Δd) || notangent(Δd.C) ? CRC.NoTangent() : noise_tangent(fx.Σy, Δd.C)
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x̄, Σy=Σ̄)
        return CRC.NoTangent(), f̄x, ȳ
    end
    return post, posterior_pullback
end

# the input gradient comes back in the test points' layout: as the training container's storage
function as_storage(xg, X, from, to)
    (X isa AbstractVector || from == to) && return xg
    return permutedims(xg)
end

function CRC.rrule(::typeof(logpdf), fx::DevPostFiniteGP{T}, Y::AbstractVecOrMat{<:Real}) where {T}
    p = fx.f
    lp = logpdf(fx, Y)
    c = ctx(); Xs, layout, D = points(fx.x); M = length(fx)
    X, xlayout, _ = points(p.data.x); N = p.data.C.n
    Ym = convert(Matrix{T}, reshape(Y, M, :)); S = size(Ym, 2)
    ms, k2 = mean_spec(p.prior.mean, fx.x, T); ns, k3 = noise_spec(fx.Σy, T)
    composite = !supported(p.prior)
    function pred_logpdf_pullback(Δ)
        Δ = CRC.unthunk(Δ)
        Δ isa CRC.AbstractZero && return CRC.NoTangent(), CRC.ZeroTangent(), CRC.ZeroTangent()
        w = convert(Vector{Float64}, Δ isa Real ? [Δ] : Δ)
        glen = composite ? ccall((:agp_post_grad_len, libagp), Int64, (Ptr{Cvoid},), p.data.C.h) : 5 + D
        g = Vector{Float64}(undef, glen); nd = Vector{T}(undef, N); ȳ = Vector{T}(undef, N)
        xg = X isa AbstractVector || xlayout == layout ? similar(X, T) : similar(permutedims(X), T)
        nsd = Vector{T}(undef, M); Ȳ = Matrix{T}(undef, M, S); xsg = similar(Xs, T)
        lock(c.lock) do
            GC.@preserve Xs Ym w g nd ȳ xg nsd Ȳ xsg k2 k3 check(c, ccall((:agp_post_pred_logpdf_grad, libagp), Int32,
                (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ref{AgpMean}, Ref{AgpNoise}, Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Cvoid},
                 Ptr{Float64}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                p.data.C.h, layout, Xs, M, ms, ns, Ym, S, w, C_NULL, g, nd, C_NULL, ȳ, xg, nsd, C_NULL, Ȳ, xsg))
        end
        # grad_out[5] is d/dc through both sides; the prior mean's tangent keeps the test side, data.δ carries the rest
        gs = (variance=g[1], scale=g[2], linear_c=g[3], noise=g[4], mean_c=g[5] + sum(ȳ), ard=g[6:end], noise_diag=nd)
        if composite
            kt = ctangent(p.prior.kernel, Int[], composite_grads(p.prior.kernel, D, g), 1.0)
        else
            _, var, _, wt = flat(p.prior.kernel)
            kt = kernel_tangent(p.prior.kernel, gs, var, wt === nothing ? 1.0 : wt)
        end
        p̄rior = CRC.Tangent{typeof(p.prior)}(; mean=mean_tangent(p.prior.mean, gs), kernel=kt)
        d̄ata = CRC.Tangent{typeof(p.data)}(; C=(noise=g[4], noise_diag=nd),
                                            x=x_tangent(p.data.x, as_storage(xg, X, layout, xlayout)), δ=ȳ)
        f̄ = CRC.Tangent{typeof(p)}(; prior=p̄rior, data=d̄ata)
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, xsg), Σy=noise_tangent(fx.Σy, (noise=sum(nsd), noise_diag=nsd)))
        return CRC.NoTangent(), f̄x, Y isa AbstractVector ? vec(Ȳ) : Ȳ
    end
    return lp, pred_logpdf_pullback
end

# ---- reverse-mode rule for rand(rng, fx, S) (test/finite_gp_projection.jl:105-127) -----------------------------------
# The forward pass draws Z exactly as the primal method above and calls agp_rand; the pullback sends the cotangent of the
# samples through ONE agp_rand_grad call at the same Z (the factor is formed again there).  The tangents reuse the logpdf
# rule's helpers; the rng gets NoTangent.  Unclaimed priors get no rule, so AD differentiates the stock method.
# A CustomMean is a closure of x (and of whatever it captures) that the engine only sees evaluated: for such a prior the
# rule differentiates `mean_split_rand` instead -- the closure's values plus a sample of the zero-mean prior, the same
# numbers as the primal method (which adds the same T-rounded mean vector to the same L Z) -- so AD takes the closure's
# own derivative with respect to x and its parameters, and only the zero-mean sample goes through agp_rand_grad.
function composite_grad_len(k, D)   # the slots composite_grads reads, in agp_post_logpdf_grad's composite layout
    n = 5
    for (_, fs) in walk(k)
        n += 1
        for (leaf, _, tr) in fs
            kind = transform_of(tr, D)[1]
            n += kind == 1 ? 1 : (kind == 2 ? D : 0)
            n += leaf isa Union{RationalQuadraticKernel,LinearKernel,ConstantKernel} ? 1 : 0
            n += leaf isa PeriodicKernel ? D : 0
        end
    end
    return n
end

mean_split_rand(rng, fx::DevFiniteGP{T}, S) where {T} =
    T.(AbstractGPs.mean_vector(fx.f.mean, fx.x)) .+ Random.rand(rng, FiniteGP(GP(AbstractGPs.ZeroMean(), fx.f.kernel), fx.x, fx.Σy), S)

function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(Random.rand), rng::Random.AbstractRNG,
                   fx::DevFiniteGP{T}, S::Int) where {T}
    claimed(fx.f) || return nothing
    fx.f.mean isa AbstractGPs.CustomMean && return CRC.rrule_via_ad(config, mean_split_rand, rng, fx, S)
    c = ctx(); X, layout, D = points(fx.x); N = length(fx); Z = randn(rng, T, N, S); out = similar(Z)
    ks, k1 = kernel_spec(fx.f.kernel, T, D); ms, k2 = mean_spec(fx.f.mean, fx.x, T); ns, k3 = noise_spec(fx.Σy, T)
    lock(c.lock) do
        GC.@preserve X k1 k2 k3 check(c, ccall((:agp_rand, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ref{AgpKernel}, Ref{AgpMean}, Ref{AgpNoise}, Int32, Ptr{Cvoid}, Int64, Int32, Ptr{Cvoid}, Int32, Ptr{Cvoid}),
            c.h, agp_dtype(T), ks, ms, ns, layout, X, N, D, Z, S, out))
    end
    composite = !supported(fx.f)
    function rand_pullback(Δ)
        Δ = CRC.unthunk(Δ)
        Δ isa CRC.AbstractZero && return CRC.NoTangent(), CRC.NoTangent(), CRC.ZeroTangent(), CRC.NoTangent()
        Ō = convert(Matrix{T}, Δ)
        g = Vector{Float64}(undef, composite ? composite_grad_len(fx.f.kernel, D) : 5 + D)
        nd = Vector{T}(undef, N); xg = similar(X, T)
        lock(c.lock) do
            GC.@preserve X Ō g nd xg k1 k2 k3 check(c, ccall((:agp_rand_grad, libagp), Int32,
                (Ptr{Cvoid}, Int32, Ref{AgpKernel}, Ref{AgpMean}, Ref{AgpNoise}, Int32, Ptr{Cvoid}, Int64, Int32, Ptr{Cvoid}, Int32,
                 Ptr{Cvoid}, Ptr{Float64}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                c.h, agp_dtype(T), ks, ms, ns, layout, X, N, D, Z, S, Ō, g, nd, C_NULL, xg, C_NULL))
        end
        gs = (variance=g[1], scale=g[2], linear_c=g[3], noise=g[4], mean_c=g[5], ard=g[6:end], noise_diag=nd)
        if composite
            kt = ctangent(fx.f.kernel, Int[], composite_grads(fx.f.kernel, D, g), 1.0)
        else
            _, var, _, w = flat(fx.f.kernel)
            kt = kernel_tangent(fx.f.kernel, gs, var, w === nothing ? 1.0 : w)
        end
        f̄ = CRC.Tangent{typeof(fx.f)}(; mean=mean_tangent(fx.f.mean, gs), kernel=kt)
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, xg), Σy=noise_tangent(fx.Σy, gs))
        return CRC.NoTangent(), CRC.NoTangent(), f̄x, CRC.NoTangent()
    end
    return out, rand_pullback
end

# ---- reverse-mode rule for rand(rng, fx, S) over a device posterior (Monte Carlo acquisition functions: q-EI, q-NEI,
# q-KG differentiate reparameterised samples μ* + L* Z with respect to x* and the hyper-parameters) --------------------
# The forward pass is the primal method's (post_rand_primal: Z from the caller's rng, then agp_post_rand); the pullback
# makes ONE agp_post_rand_grad call at the same Z.  The tangents are those of the logpdf-over-posterior rule: the kernel, data.x,
# data.δ = ȳ and data.C in the DevPosterior's tangent (the posterior rule routes them on), the test points, noise and
# the prior mean's test side in fx's.  A CustomMean prior goes through AD of `mean_split_post_rand`: the closure's values
# at x* plus a device sample with a zero test mean (`zero_mean_post_rand`, whose rule is the same pullback).
function post_rand_primal(rng, fx::DevPostFiniteGP{T}, S::Int, zero_mean::Bool) where {T}
    p = fx.f; c = ctx(); Xs, layout, D = points(fx.x); M = length(fx)
    Z = randn(rng, T, M, S); out = similar(Z)
    ms, k2 = zero_mean ? mean_spec(AbstractGPs.ZeroMean(), fx.x, T) : mean_spec(p.prior.mean, fx.x, T)
    ns, k3 = noise_spec(fx.Σy, T)
    lock(c.lock) do
        GC.@preserve Xs k2 k3 check(c, ccall((:agp_post_rand, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ref{AgpMean}, Ref{AgpNoise}, Ptr{Cvoid}, Int32, Ptr{Cvoid}),
            p.data.C.h, layout, Xs, M, ms, ns, Z, S, out))
    end
    return out, Z, ms, k2, ns, k3
end

zero_mean_post_rand(rng, fx::DevPostFiniteGP, S::Int) = post_rand_primal(rng, fx, S, true)[1]
mean_split_post_rand(rng, fx::DevPostFiniteGP{T}, S::Int) where {T} =
    T.(AbstractGPs.mean_vector(fx.f.prior.mean, fx.x)) .+ zero_mean_post_rand(rng, fx, S)

function post_rand_rrule(rng, fx::DevPostFiniteGP{T}, S::Int, zero_mean::Bool) where {T}
    p = fx.f
    out, Z, ms, k2, ns, k3 = post_rand_primal(rng, fx, S, zero_mean)
    c = ctx(); Xs, layout, D = points(fx.x); M = length(fx)
    X, xlayout, _ = points(p.data.x); N = p.data.C.n
    composite = !supported(p.prior)
    function post_rand_pullback(Δ)
        Δ = CRC.unthunk(Δ)
        Δ isa CRC.AbstractZero && return CRC.NoTangent(), CRC.NoTangent(), CRC.ZeroTangent(), CRC.NoTangent()
        Ō = convert(Matrix{T}, Δ)
        glen = composite ? ccall((:agp_post_grad_len, libagp), Int64, (Ptr{Cvoid},), p.data.C.h) : 5 + D
        g = Vector{Float64}(undef, glen); nd = Vector{T}(undef, N); ȳ = Vector{T}(undef, N)
        xg = X isa AbstractVector || xlayout == layout ? similar(X, T) : similar(permutedims(X), T)
        nsd = Vector{T}(undef, M); xsg = similar(Xs, T)
        lock(c.lock) do
            GC.@preserve Xs Z Ō g nd ȳ xg nsd xsg k2 k3 check(c, ccall((:agp_post_rand_grad, libagp), Int32,
                (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ref{AgpMean}, Ref{AgpNoise}, Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Float64},
                 Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                p.data.C.h, layout, Xs, M, ms, ns, Z, S, Ō, g, nd, C_NULL, ȳ, xg, nsd, C_NULL, C_NULL, xsg))
        end
        # grad_out[5] is d/dc through both sides; the prior mean's tangent keeps the test side, data.δ carries the rest
        gs = (variance=g[1], scale=g[2], linear_c=g[3], noise=g[4], mean_c=g[5] + sum(ȳ), ard=g[6:end], noise_diag=nd)
        if composite
            kt = ctangent(p.prior.kernel, Int[], composite_grads(p.prior.kernel, D, g), 1.0)
        else
            _, var, _, wt = flat(p.prior.kernel)
            kt = kernel_tangent(p.prior.kernel, gs, var, wt === nothing ? 1.0 : wt)
        end
        m̄ = zero_mean ? CRC.NoTangent() : mean_tangent(p.prior.mean, gs)
        p̄rior = CRC.Tangent{typeof(p.prior)}(; mean=m̄, kernel=kt)
        d̄ata = CRC.Tangent{typeof(p.data)}(; C=(noise=g[4], noise_diag=nd),
                                            x=x_tangent(p.data.x, as_storage(xg, X, layout, xlayout)), δ=ȳ)
        f̄ = CRC.Tangent{typeof(p)}(; prior=p̄rior, data=d̄ata)
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, xsg), Σy=noise_tangent(fx.Σy, (noise=sum(nsd), noise_diag=nsd)))
        return CRC.NoTangent(), CRC.NoTangent(), f̄x, CRC.NoTangent()
    end
    return out, post_rand_pullback
end

function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(Random.rand), rng::Random.AbstractRNG,
                   fx::DevPostFiniteGP{T}, S::Int) where {T}
    fx.f.prior.mean isa AbstractGPs.CustomMean && return CRC.rrule_via_ad(config, mean_split_post_rand, rng, fx, S)
    return post_rand_rrule(rng, fx, S, false)
end
CRC.rrule(::typeof(zero_mean_post_rand), rng::Random.AbstractRNG, fx::DevPostFiniteGP, S::Int) =
    post_rand_rrule(rng, fx, S, true)

# ---- reverse-mode rule for mean_and_var over a device posterior (analytic acquisition functions: expected improvement,
# probability of improvement and UCB are closed forms in μ(x*) and σ²(x*), maximised over x*; marginals goes through it)
# The forward pass is the primal method's (post_mean_var_primal, agp_post_mean_var); the pullback makes ONE
# agp_post_mean_var_grad call with every output at the cotangents (m̄, v̄).  The tangents are those of the rand-over-posterior
# rule: the kernel, data.x, data.δ = ȳ and data.C in the DevPosterior's tangent (the posterior rule routes them on); fx.x
# gets the x* gradient and fx.Σy Diagonal(v̄), since the test noise adds to the variances.  A CustomMean prior goes through
# AD of `mean_split_post_mean_var`: the closure's values at x* plus the device means and variances under a zero test mean
# (`zero_mean_post_mean_var`, whose rule is the same pullback).
zero_mean_post_mean_var(fx::DevPostFiniteGP) = post_mean_var_primal(fx, true)
function mean_split_post_mean_var(fx::DevPostFiniteGP{T}) where {T}
    μ0, v = zero_mean_post_mean_var(fx)
    return T.(AbstractGPs.mean_vector(fx.f.prior.mean, fx.x)) .+ μ0, v
end

function post_mean_var_rrule(fx::DevPostFiniteGP{T}, zero_mean::Bool) where {T}
    p = fx.f
    μ, v = post_mean_var_primal(fx, zero_mean)
    c = ctx(); Xs, layout, D = points(fx.x); M = length(fx)
    X, xlayout, _ = points(p.data.x); N = p.data.C.n
    composite = !supported(p.prior)
    function post_mean_var_pullback(Δ)
        Δ = CRC.unthunk(Δ)
        Δ isa CRC.AbstractZero && return CRC.NoTangent(), CRC.ZeroTangent()
        m̄ = notangent(Δ[1]) ? zeros(T, M) : convert(Vector{T}, CRC.unthunk(Δ[1]))
        v̄ = notangent(Δ[2]) ? zeros(T, M) : convert(Vector{T}, CRC.unthunk(Δ[2]))
        glen = composite ? ccall((:agp_post_grad_len, libagp), Int64, (Ptr{Cvoid},), p.data.C.h) : 5 + D
        g = Vector{Float64}(undef, glen); nd = Vector{T}(undef, N); ȳ = Vector{T}(undef, N)
        xg = X isa AbstractVector || xlayout == layout ? similar(X, T) : similar(permutedims(X), T)
        xsg = similar(Xs, T)
        lock(c.lock) do
            GC.@preserve Xs m̄ v̄ g nd ȳ xg xsg check(c, ccall((:agp_post_mean_var_grad, libagp), Int32,
                (Ptr{Cvoid}, Int32, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Float64}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid},
                 Ptr{Cvoid}, Ptr{Cvoid}),
                p.data.C.h, layout, Xs, M, m̄, v̄, g, nd, C_NULL, ȳ, xg, xsg))
        end
        # grad_out[5] is d/dc through both sides; the prior mean's tangent keeps the test side, data.δ carries the rest
        gs = (variance=g[1], scale=g[2], linear_c=g[3], noise=g[4], mean_c=g[5] + sum(ȳ), ard=g[6:end], noise_diag=nd)
        if composite
            kt = ctangent(p.prior.kernel, Int[], composite_grads(p.prior.kernel, D, g), 1.0)
        else
            _, var, _, wt = flat(p.prior.kernel)
            kt = kernel_tangent(p.prior.kernel, gs, var, wt === nothing ? 1.0 : wt)
        end
        mt = zero_mean ? CRC.NoTangent() : mean_tangent(p.prior.mean, gs)
        p̄rior = CRC.Tangent{typeof(p.prior)}(; mean=mt, kernel=kt)
        d̄ata = CRC.Tangent{typeof(p.data)}(; C=(noise=g[4], noise_diag=nd),
                                            x=x_tangent(p.data.x, as_storage(xg, X, layout, xlayout)), δ=ȳ)
        f̄ = CRC.Tangent{typeof(p)}(; prior=p̄rior, data=d̄ata)
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, xsg), Σy=noise_tangent(fx.Σy, (noise=sum(v̄), noise_diag=v̄)))
        return CRC.NoTangent(), f̄x
    end
    return (μ, v), post_mean_var_pullback
end

function CRC.rrule(config::CRC.RuleConfig{>:CRC.HasReverseMode}, ::typeof(mean_and_var), fx::DevPostFiniteGP{T}) where {T}
    fx.f.prior.mean isa AbstractGPs.CustomMean && return CRC.rrule_via_ad(config, mean_split_post_mean_var, fx)
    return post_mean_var_rrule(fx, false)
end
CRC.rrule(::typeof(zero_mean_post_mean_var), fx::DevPostFiniteGP) = post_mean_var_rrule(fx, true)

# ---- reverse-mode rules for the VFE objectives: elbo(VFE(fz), fx, y) and approx_log_evidence(VFE | DTC, fx, y) ---------
# (src/sparse_approximations.jl:248-254, :282-286).  One agp_vfe_elbo_grad_x call returns the value, the kernel / noise /
# mean gradients in agp_post_logpdf_grad's layout (mapped back by the logpdf rule's helpers), the per-point noise and mean
# gradients and the gradients with respect to the inducing points and the training inputs.  The kernel's tangent goes to
# fx.f (fz.f is the same GP); fz receives the tangent of its inputs only, not of its jitter; fx.x receives the tangent of
# its inputs, so a feature network that computes x learns from the GP term (the mean and per-point noise are taken as
# constants of x, agp.h).
z_storage(z::ColVecs, zg, layout) = layout == AGP_POINT_MAJOR ? zg : permutedims(zg)
z_storage(z::RowVecs, zg, layout) = layout == AGP_FEATURE_MAJOR ? zg : permutedims(zg)
z_storage(z::AbstractVector{<:Real}, zg, layout) = zg

function sparse_gradients(fz::FiniteGP, fx::DevFiniteGP{T}, y::AbstractVector{<:Real}, objective) where {T}
    fz.f === fx.f || throw(ArgumentError("the inducing and the data FiniteGP must share the prior"))
    length(y) == length(fx) || throw(DimensionMismatch("length(fx) = $(length(fx)) but length(y) = $(length(y))"))
    c = ctx(); X, layout, D = points(fx.x); Z = same_layout(fz.x, layout)
    ks, k1 = kernel_spec(fx.f.kernel, T); ms, k2 = mean_spec(fx.f.mean, fx.x, T)
    ns, k3 = noise_spec(fx.Σy, T); js, k4 = noise_spec(fz.Σy, T)
    yv = convert(Vector{T}, y); val = Vector{T}(undef, 1); g = Vector{Float64}(undef, 5 + D)
    nd = Vector{T}(undef, length(fx)); md = Vector{T}(undef, length(fx)); zg = similar(Z, T); xg = similar(X, T)
    lock(c.lock) do
        GC.@preserve X Z yv val g nd md zg xg k1 k2 k3 k4 check(c, ccall((:agp_vfe_elbo_grad_x, libagp), Int32,
            (Ptr{Cvoid}, Int32, Ref{AgpKernel}, Ref{AgpMean}, Ref{AgpNoise}, Int32, Ptr{Cvoid}, Int64, Int32, Ptr{Cvoid}, Int64,
             Ref{AgpNoise}, Ptr{Cvoid}, Int32, Ptr{Cvoid}, Ptr{Float64}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
            c.h, agp_dtype(T), ks, ms, ns, layout, X, length(fx), D, Z, length(fz), js, yv, Int32(objective), val, g, nd, md, zg,
            xg))
    end
    return val[1], g, nd, md, z_storage(fz.x, zg, layout), xg
end

function vfe_rrule(approx, fx::DevFiniteGP{T}, y::AbstractVector{<:Real}) where {T}
    fz = approx.fz
    val, gv, nd, md, zg, xg = sparse_gradients(fz, fx, y, approx isa DTC ? 1 : 0)
    g = (variance=gv[1], scale=gv[2], linear_c=gv[3], noise=gv[4], mean_c=gv[5], ard=gv[6:end], noise_diag=nd)
    _, var, _, w = flat(fx.f.kernel)
    w === nothing && (w = 1.0)
    function vfe_pullback(Δ)
        d = CRC.unthunk(Δ)
        gs = map(v -> v isa Number ? d * v : d .* v, g)
        f̄ = CRC.Tangent{typeof(fx.f)}(; mean=mean_tangent(fx.f.mean, gs), kernel=kernel_tangent(fx.f.kernel, gs, var, w))
        f̄x = CRC.Tangent{typeof(fx)}(; f=f̄, x=x_tangent(fx.x, d .* xg), Σy=noise_tangent(fx.Σy, gs))
        t_approx = CRC.Tangent{typeof(approx)}(; fz=CRC.Tangent{typeof(fz)}(; x=x_tangent(fz.x, d .* zg)))
        return CRC.NoTangent(), t_approx, f̄x, -d .* md                    # d/d y = -d/d m
    end
    return val, vfe_pullback
end

CRC.rrule(::typeof(elbo), vfe::VFE, fx::DevFiniteGP, y::AbstractVector{<:Real}) =
    supported(fx.f) ? vfe_rrule(vfe, fx, y) : nothing
CRC.rrule(::typeof(approx_log_evidence), approx::Union{VFE,DTC}, fx::DevFiniteGP, y::AbstractVector{<:Real}) =
    supported(fx.f) ? vfe_rrule(approx, fx, y) : nothing

end # module
