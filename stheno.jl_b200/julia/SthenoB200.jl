# SthenoB200.jl -- thin `ccall` shim that routes Stheno/AbstractGPs' dense-GP hot path to
# libstheno_b200.so (include/stheno_b200.h).
#
# STATUS: written against Stheno v0.8.2 / AbstractGPs 0.5 / KernelFunctions 0.10; it has NOT been
# executed (no `julia` binary in the build image or on the GPU box).  What IS checked mechanically
# (tests/test_julia_shim.py, CPU): every `ccall` in this file names an exported symbol, passes the
# number of arguments the C prototype declares with compatible types, and every `struct Sb*` has
# the field order / types of its C twin.  The Python mirror stheno.jl_b200/{gp,finite,lib}.py binds
# the same symbols call for call and is what the tests and the benchmark run.
#
# Usage
#     using Stheno, SthenoB200
#     f  = @gppp let f1 = GP(SEKernel()); f2 = GP(Matern52Kernel()); f3 = f1 + f2 end
#     fb = b200(f)                                  # device-marked programme
#     fx = fb(BlockData(GPPPInput(:f1, x1), GPPPInput(:f3, x3)), 0.1)
#     logpdf(fx, y); fp = posterior(fx, y); mean_and_var(fp(GPPPInput(:f2, xs)))
#     elbo(VFE(fb(GPPPInput(:f3, z), 1e-9)), fx, y)
module SthenoB200

using Stheno, AbstractGPs, KernelFunctions, LinearAlgebra, Random
using Stheno: AtomicGP, DerivedGP, GPPP, BlockData, GPPPInput, SthenoAbstractGP, SparseFiniteGP
import AbstractGPs: logpdf, posterior, mean, var, cov, mean_and_var, mean_and_cov, marginals, rand, elbo, dtc
import Statistics
import Distributions: Normal

const LIB = get(ENV, "STHENO_B200_LIB", "libstheno_b200.so")

# ---- C structs (layout == include/stheno_b200.h) ---------------------------------------------
struct SbArray
    data::Ptr{Cvoid}; n::Int64; dim::Int32; reserved::Int32
end
struct SbTerm
    kernel::Int32; zl::Int32; zr::Int32; sl::Int32; sr::Int32; reserved::Int32
    coeff::Float64; param::Float64
end
struct SbBlock
    row0::Int64; nrows::Int64; col0::Int64; ncols::Int64; term0::Int32; nterms::Int32
end
struct SbCovSpec
    nrows::Int64; ncols::Int64; symmetric::Int32; narrays::Int32; arrays::Ptr{SbArray}
    nterms::Int32; terms::Ptr{SbTerm}; nblocks::Int32; blocks::Ptr{SbBlock}
end
struct SbNoise
    sigma2::Float64; diag::Ptr{Cvoid}; dense::Ptr{Cvoid}
end

const K_SE, K_M12, K_M32, K_M52, K_WHITE, K_CONST = Int32.(0:5)

function check(status::Int32, info::Int64=0)
    status == 0 && return
    msg = unsafe_string(ccall((:sb_last_error, LIB), Cstring, ()))
    status == -3 && throw(LinearAlgebra.PosDefException(info))   # what `cholesky` throws
    status == -4 && error("SthenoB200: unsupported: $msg")
    status == -1 && throw(ArgumentError(msg))
    error("SthenoB200 (status $status): $msg")
end

# ---- context / handles ------------------------------------------------------------------------
mutable struct Context
    h::Ptr{Cvoid}
    function Context(device::Integer=0)
        r = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:sb_ctx_create, LIB), Int32, (Int32, Ref{Ptr{Cvoid}}), device, r))
        c = new(r[])
        finalizer(c -> ccall((:sb_ctx_destroy, LIB), Int32, (Ptr{Cvoid},), c.h), c)
        c
    end
end
const CTX = Ref{Union{Nothing,Context}}(nothing)
ctx() = (CTX[] === nothing && (CTX[] = Context()); CTX[])

mutable struct Factor
    h::Ptr{Cvoid}
    n::Int
    alpha_owner::Any     # the posterior whose alpha currently sits in the device handle
end
function destroy!(F::Factor)
    F.h != C_NULL && ccall((:sb_factor_destroy, LIB), Int32, (Ptr{Cvoid},), F.h)
    F.h = C_NULL
end
mutable struct VfeHandle
    h::Ptr{Cvoid}
end
function destroy!(V::VfeHandle)
    V.h != C_NULL && ccall((:sb_vfe_destroy, LIB), Int32, (Ptr{Cvoid},), V.h)
    V.h = C_NULL
end

# ---- plan lowering (SURVEY App. B.3): process -> mean vector, [(atom, coeff, scale, z, key)] ----
# key = ids of the chain of wrapping atomics when a whole GPPP is used as an atomic inside another
# programme (test/gaussian_process_probabilistic_programme.jl:107-120): two different outer atomics
# wrapping the same inner programme are independent.
struct LTerm
    atom::AtomicGP; coeff::Float64; scale::Union{Nothing,Vector{Float64}}; z; key::Tuple
end
same_leaf(a::LTerm, b::LTerm) = a.atom === b.atom && a.key == b.key      # atomic_gp.jl:36-38

function lower(f::AtomicGP, x)
    if f.gp isa GPPP                                   # nested programme: x is a GPPPInput of the inner one
        x isa GPPPInput || error("SthenoB200: nested GPPP needs GPPPInput inner inputs")
        m, t = lower(f.gp.fs[x.p], x.x)
        return m, [LTerm(u.atom, u.coeff, u.scale, u.z, (objectid(f), u.key...)) for u in t]
    end
    return AbstractGPs.mean_vector(f.gp.mean, x), [LTerm(f, 1.0, nothing, x, ())]
end
function lower(f::DerivedGP, x)
    op = f.args[1]
    if op === (+) && f.args[2] isa AbstractGPs.AbstractGP          # addition.jl:26-47
        ma, ta = lower(f.args[2], x); mb, tb = lower(f.args[3], x)
        return ma .+ mb, vcat(ta, tb)
    elseif op === (+)                                              # addition.jl:73-86 (known)
        b = f.args[2]; m, t = lower(f.args[3], x)
        return (b isa Real ? b .+ m : b.(x) .+ m), t
    elseif op === (*)                                              # product.jl:25-70
        s = f.args[2]; m, t = lower(f.args[3], x)
        if s isa Real
            return s .* m, [LTerm(u.atom, s * u.coeff, u.scale, u.z, u.key) for u in t]
        end
        sx = Float64.(s.(x))
        return sx .* m, [LTerm(u.atom, u.coeff, u.scale === nothing ? sx : sx .* u.scale, u.z, u.key) for u in t]
    elseif op === (∘)                                              # compose.jl:16-28
        return lower(f.args[2], f.args[3].(x))
    end
    error("SthenoB200: cannot lower $(op)")
end

# kernel -> [(coeff, id, param, input scale)]
klower(::SEKernel) = [(1.0, K_SE, 0.0, 1.0)]
klower(::Matern12Kernel) = [(1.0, K_M12, 0.0, 1.0)]
klower(::Matern32Kernel) = [(1.0, K_M32, 0.0, 1.0)]
klower(::Matern52Kernel) = [(1.0, K_M52, 0.0, 1.0)]
klower(::WhiteKernel) = [(1.0, K_WHITE, 0.0, 1.0)]
klower(k::ConstantKernel) = [(1.0, K_CONST, Float64(only(k.c)), 1.0)]
klower(k::ScaledKernel) = [(c * only(k.σ²), id, p, s) for (c, id, p, s) in klower(k.kernel)]
klower(k::KernelSum) = reduce(vcat, klower.(k.kernels))
klower(k::TransformedKernel{<:Any,<:ScaleTransform}) =
    [(c, id, p, s * only(k.transform.s)) for (c, id, p, s) in klower(k.kernel)]

pointmajor(z::AbstractVector{<:Real}, s) = reshape(Float64.(z) .* s, 1, :)   # 1 x n  (dim 1)
pointmajor(z::ColVecs, s) = Float64.(z.X) .* s                               # D x n  == point-major

# Spec builder.  which = :sym  lower block triangle (factor path), :all every (i, j) block,
# :diag only the paired (i, i) blocks (var(f, x): cross.jl:64-67; the library evaluates a diag
# block elementwise, point i with point i).  `keep` holds every Julia array the pointers refer to
# (GC.@preserve keep ... around the ccall).
function build_spec(procs_r, xs_r, procs_c, xs_c; which::Symbol)
    arrays = SbArray[]; terms = SbTerm[]; blocks = SbBlock[]; keep = Any[]
    cache = IdDict{Any,Dict{Float64,Int32}}()
    function push_arr!(a::Matrix{Float64}, dim)
        push!(keep, a); push!(arrays, SbArray(pointer(a), size(a, 2), dim, 0)); Int32(length(arrays) - 1)
    end
    function input!(z, s)                                # one upload per (input collection, scale)
        d = get!(cache, z, Dict{Float64,Int32}())
        get!(d, s) do
            a = pointmajor(z, s); push_arr!(a, size(a, 1))
        end
    end
    push_scale!(s) = s === nothing ? Int32(-1) : push_arr!(reshape(s, 1, :), 0)
    lr = [lower(p, x)[2] for (p, x) in zip(procs_r, xs_r)]
    lc = (procs_c === procs_r && xs_c === xs_r) ? lr : [lower(p, x)[2] for (p, x) in zip(procs_c, xs_c)]
    r0 = cumsum([0; length.(xs_r)]); c0 = cumsum([0; length.(xs_c)])
    for i in eachindex(procs_r), j in eachindex(procs_c)
        which === :sym && j > i && continue
        which === :diag && j != i && continue
        t0 = length(terms)
        for a in lr[i], b in lc[j]
            same_leaf(a, b) || continue                              # independent leaves: zeros
            for (kc, id, p, s) in klower(a.atom.gp.kernel)
                push!(terms, SbTerm(id, input!(a.z, s), input!(b.z, s), push_scale!(a.scale), push_scale!(b.scale),
                                    0, a.coeff * b.coeff * kc, p))
            end
        end
        push!(blocks, SbBlock(r0[i], length(xs_r[i]), c0[j], length(xs_c[j]), t0, length(terms) - t0))
    end
    push!(keep, arrays, terms, blocks)
    spec = SbCovSpec(r0[end], c0[end], which === :sym ? 1 : 0, length(arrays), pointer(arrays), length(terms),
                     pointer(terms), length(blocks), pointer(blocks))
    return spec, keep
end

# ---- device-marked programme and the AbstractGPs methods it overrides ---------------------------
struct B200GPPP{T<:GPPP} <: AbstractGPs.AbstractGP
    f::T
end
b200(f::GPPP) = B200GPPP(f)

# extract_components (gppp.jl:25, 27-30, 32-43) without allocating a `cross` node
components(f::B200GPPP, x::GPPPInput) = (Any[f.f.fs[x.p]], Any[x.x])
function components(f::B200GPPP, x::BlockData)
    ps = Any[]; vs = Any[]
    for b in x.X
        p, v = components(f, b); append!(ps, p); append!(vs, v)
    end
    ps, vs
end
function components(f::B200GPPP, x::AbstractVector{<:Tuple{Symbol,Any}})   # gppp.jl:32-43: regroup by symbol
    syms = first.(x); feats = last.(x)
    blocks = [GPPPInput(s, _stack(feats[findall(==(s), syms)])) for s in unique(syms)]
    components(f, BlockData(blocks))
end
_stack(v::AbstractVector{<:Real}) = collect(Float64, v)
_stack(v::AbstractVector{<:AbstractVector}) = ColVecs(reduce(hcat, v))

npoints(x) = length(x)
lowered_mean(f::B200GPPP, x) = reduce(vcat, [lower(p, v)[1] for (p, v) in zip(components(f, x)...)])

# internal AbstractGPs API on the marked programme (docs/src/internals.md:8-24): parity / small N
mean(f::B200GPPP, x::AbstractVector) = lowered_mean(f, x)
function cov(f::B200GPPP, x::AbstractVector, y::AbstractVector=x)
    pr, vr = components(f, x); pc, vc = x === y ? (pr, vr) : components(f, y)
    spec, keep = build_spec(pr, vr, pc, vc; which=:all)
    K = Matrix{Float64}(undef, npoints(x), npoints(y))
    GC.@preserve keep K check(ccall((:sb_cov_dense, LIB), Int32, (Ptr{Cvoid}, Ref{SbCovSpec}, Ptr{Cvoid}),
                                    ctx().h, spec, K))
    K
end
function var(f::B200GPPP, x::AbstractVector, y::AbstractVector=x)
    pr, vr = components(f, x); pc, vc = x === y ? (pr, vr) : components(f, y)
    spec, keep = build_spec(pr, vr, pc, vc; which=:diag)
    v = Vector{Float64}(undef, npoints(x))
    GC.@preserve keep v check(ccall((:sb_cov_diag, LIB), Int32, (Ptr{Cvoid}, Ref{SbCovSpec}, Ptr{Cvoid}),
                                    ctx().h, spec, v))
    v
end
mean_and_cov(f::B200GPPP, x::AbstractVector) = (mean(f, x), cov(f, x))
mean_and_var(f::B200GPPP, x::AbstractVector) = (mean(f, x), var(f, x))

const B200Finite = AbstractGPs.FiniteGP{<:B200GPPP}
host_mean(fx::B200Finite) = lowered_mean(fx.f, fx.x)

# Sigma_y -> sb_noise: isotropic (Fill diagonal) = scalar fast path, Diagonal, or dense PSD
function noise_struct(Σ)
    if Σ isa Diagonal && all(==(first(Σ.diag)), Σ.diag)
        return SbNoise(Float64(first(Σ.diag)), C_NULL, C_NULL), nothing
    elseif Σ isa Diagonal
        nd = collect(Float64, Σ.diag)
        return SbNoise(0.0, pointer(nd), C_NULL), nd
    end
    nd = Matrix{Float64}(Σ)
    return SbNoise(0.0, C_NULL, pointer(nd)), nd
end

function factor(fx::B200Finite)
    ps, vs = components(fx.f, fx.x)
    spec, keep = build_spec(ps, vs, ps, vs; which=:sym)
    noise, nd = noise_struct(fx.Σy)
    h = Ref{Ptr{Cvoid}}(C_NULL); info = Ref{Int64}(0)
    st = GC.@preserve keep nd ccall((:sb_factor_create, LIB), Int32,
        (Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbNoise}, Ref{Ptr{Cvoid}}, Ref{Int64}), ctx().h, spec, noise, h, info)
    check(st, info[])
    F = Factor(h[], npoints(fx.x), nothing); finalizer(destroy!, F); F
end

function logpdf(fx::B200Finite, Y::AbstractVecOrMat{<:Real})
    F = factor(fx)
    δ = Matrix{Float64}(reshape(Y, size(Y, 1), :) .- host_mean(fx)); S = size(δ, 2)
    out = Vector{Float64}(undef, S)
    GC.@preserve δ out check(ccall((:sb_logpdf, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int32, Ptr{Float64}), ctx().h, F.h, δ, S, out))
    Y isa AbstractVector ? out[1] : out
end

cov(fx::B200Finite) = cov(fx.f, fx.x) + fx.Σy
cov(fx::B200Finite, gx::B200Finite) = cov(fx.f, fx.x, gx.x)          # src/gp/util.jl:12-14
var(fx::B200Finite) = var(fx.f, fx.x) .+ diag(fx.Σy)
mean(fx::B200Finite) = host_mean(fx)
marginals(fx::B200Finite) = Normal.(mean(fx), sqrt.(var(fx)))

function rand(rng::AbstractRNG, fx::B200Finite, S::Int)
    F = factor(fx); z = randn(rng, npoints(fx.x), S); out = similar(z)
    GC.@preserve z out check(ccall((:sb_rand, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int32, Ptr{Cvoid}), ctx().h, F.h, z, S, out))
    out .+ host_mean(fx)
end
rand(rng::AbstractRNG, fx::B200Finite) = vec(rand(rng, fx, 1))

# ---- exact posterior ------------------------------------------------------------------------------
struct B200PosteriorGP{T<:B200GPPP} <: AbstractGPs.AbstractGP
    prior::T; x; F::Factor; α::Vector{Float64}; δ::Vector{Float64}
end

# alpha = C \ δ on the device, stored with the factor it belongs to
function posterior_from(f::B200GPPP, x, F::Factor, δ::Vector{Float64})
    α = similar(δ)
    GC.@preserve δ check(ccall((:sb_factor_set_data, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), ctx().h, F.h, δ))
    GC.@preserve α check(ccall((:sb_factor_alpha, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), ctx().h, F.h, α))
    fp = B200PosteriorGP(f, x, F, α, δ); F.alpha_owner = fp; fp
end

posterior(fx::B200Finite, y::AbstractVector{<:Real}) = posterior_from(fx.f, fx.x, factor(fx), Float64.(y .- host_mean(fx)))

# `posterior` is pure in the reference: a posterior sharing its factor re-installs ITS alpha
function install_alpha!(fp::B200PosteriorGP)
    fp.F.alpha_owner === fp && return
    α = fp.α
    GC.@preserve α check(ccall((:sb_factor_set_alpha, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), ctx().h, fp.F.h, α))
    fp.F.alpha_owner = fp
end

function mean_and_var(fp::B200PosteriorGP, xs::AbstractVector)
    ps, vs = components(fp.prior, xs); po, vo = components(fp.prior, fp.x)
    cross, k1 = build_spec(ps, vs, po, vo; which=:all)
    pd, k2 = build_spec(ps, vs, ps, vs; which=:diag)        # paired points: only the (i, i) blocks
    n = npoints(xs); m = zeros(n); v = zeros(n)
    install_alpha!(fp)
    GC.@preserve k1 k2 m v check(ccall((:sb_predict, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ptr{Cvoid}, Ptr{Cvoid}),
        ctx().h, fp.F.h, cross, pd, m, v))
    m .+ lowered_mean(fp.prior, xs), v
end
mean(fp::B200PosteriorGP, xs::AbstractVector) = mean_and_var(fp, xs)[1]
var(fp::B200PosteriorGP, xs::AbstractVector) = mean_and_var(fp, xs)[2]

function cov(fp::B200PosteriorGP, xs::AbstractVector)
    ps, vs = components(fp.prior, xs); po, vo = components(fp.prior, fp.x)
    cross, k1 = build_spec(ps, vs, po, vo; which=:all)
    full, k2 = build_spec(ps, vs, ps, vs; which=:all)
    n = npoints(xs); K = Matrix{Float64}(undef, n, n)
    GC.@preserve k1 k2 K check(ccall((:sb_predict_cov, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ptr{Cvoid}), ctx().h, fp.F.h, cross, full, K))
    K
end
# cov(f_post, x, z) = K(x,z) - (C.U'\K_{X,x})'(C.U'\K_{X,z}): off-diagonal block of the joint posterior
function cov(fp::B200PosteriorGP, xs::AbstractVector, zs::AbstractVector)
    K = cov(fp, BlockData([xs, zs])); nx = npoints(xs)
    K[1:nx, nx+1:end]
end
mean_and_cov(fp::B200PosteriorGP, xs::AbstractVector) = (mean(fp, xs), cov(fp, xs))

const B200PostFinite = AbstractGPs.FiniteGP{<:B200PosteriorGP}
mean(fx::B200PostFinite) = mean(fx.f, fx.x)
var(fx::B200PostFinite) = var(fx.f, fx.x) .+ diag(fx.Σy)
cov(fx::B200PostFinite) = cov(fx.f, fx.x) + fx.Σy
function mean_and_var(fx::B200PostFinite)
    m, v = mean_and_var(fx.f, fx.x); m, v .+ diag(fx.Σy)
end
marginals(fx::B200PostFinite) = Normal.(mean_and_var(fx)[1], sqrt.(mean_and_var(fx)[2]))

# cholesky(cov(f_post(x*, noise))) on the device: rand / logpdf of a posterior FiniteGP (README.md:96)
function factor(fx::B200PostFinite)
    fp = fx.f
    ps, vs = components(fp.prior, fx.x); po, vo = components(fp.prior, fp.x)
    cross, k1 = build_spec(ps, vs, po, vo; which=:all)
    full, k2 = build_spec(ps, vs, ps, vs; which=:all)
    noise, nd = noise_struct(fx.Σy)
    h = Ref{Ptr{Cvoid}}(C_NULL); info = Ref{Int64}(0)
    st = GC.@preserve k1 k2 nd ccall((:sb_predict_factor, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ref{SbNoise}, Ref{Ptr{Cvoid}}, Ref{Int64}),
        ctx().h, fp.F.h, cross, full, noise, h, info)
    check(st, info[])
    F = Factor(h[], npoints(fx.x), nothing); finalizer(destroy!, F); F
end
function rand(rng::AbstractRNG, fx::B200PostFinite, S::Int)
    F = factor(fx); z = randn(rng, npoints(fx.x), S); out = similar(z)
    GC.@preserve z out check(ccall((:sb_rand, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int32, Ptr{Cvoid}), ctx().h, F.h, z, S, out))
    out .+ mean(fx)
end
rand(rng::AbstractRNG, fx::B200PostFinite) = vec(rand(rng, fx, 1))

# posterior(f_post(x2, Σ2), y2): the posterior of the stacked observations [x; x2] with block-diagonal noise.
# As AbstractGPs' update_chol, fp's factor is extended on the device (its full block columns are kept), not
# refactorised; fp itself is unchanged.
function posterior(fx::B200PostFinite, y::AbstractVector{<:Real})
    fp = fx.f
    length(y) == npoints(fx.x) || throw(DimensionMismatch("length(y) != length(fx)"))
    ps, vs = components(fp.prior, fx.x); po, vo = components(fp.prior, fp.x)
    cross, k1 = build_spec(ps, vs, po, vo; which=:all)
    full, k2 = build_spec(ps, vs, ps, vs; which=:all)
    noise, nd = noise_struct(fx.Σy)
    h = Ref{Ptr{Cvoid}}(C_NULL); info = Ref{Int64}(0)
    st = GC.@preserve k1 k2 nd ccall((:sb_factor_append, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ref{SbNoise}, Ref{Ptr{Cvoid}}, Ref{Int64}),
        ctx().h, fp.F.h, cross, full, noise, h, info)
    check(st, info[])
    x = BlockData([fp.x, fx.x])
    F = Factor(h[], npoints(x), nothing); finalizer(destroy!, F)
    posterior_from(fp.prior, x, F, vcat(fp.δ, Float64.(y .- lowered_mean(fp.prior, fx.x))))
end

function logpdf(fx::B200PostFinite, y::AbstractVector{<:Real})
    F = factor(fx); δ = Float64.(y .- mean(fx)); out = Ref{Float64}(0.0)
    GC.@preserve δ check(ccall((:sb_logpdf, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int32, Ref{Float64}), ctx().h, F.h, δ, 1, out))
    out[]
end

# ---- VFE / elbo / SparseFiniteGP (src/gp/sparse_finite_gp.jl:52-62) ---------------------------------
struct B200ApproxPosteriorGP{T<:B200GPPP} <: AbstractGPs.AbstractGP
    prior::T; z; V::VfeHandle
end

function vfe_create(fz::B200Finite, fx::B200Finite, y::AbstractVector{<:Real})
    fz.f === fx.f || throw(ArgumentError("VFE: inducing and observed FiniteGPs must share the prior"))
    length(y) == npoints(fx.x) || throw(DimensionMismatch("length(y) != length(fx)"))
    fx.Σy isa Diagonal || error("SthenoB200: VFE needs diagonal observation noise")
    pz, vz = components(fz.f, fz.x); px, vx = components(fx.f, fx.x)
    uu, k1 = build_spec(pz, vz, pz, vz; which=:sym)
    xu, k2 = build_spec(px, vx, pz, vz; which=:all)
    ffd, k3 = build_spec(px, vx, px, vx; which=:diag)
    nu, ndu = noise_struct(fz.Σy); nf, ndf = noise_struct(fx.Σy)
    δ = Float64.(y .- host_mean(fx))
    h = Ref{Ptr{Cvoid}}(C_NULL); out2 = zeros(2); info = Ref{Int64}(0)
    st = GC.@preserve k1 k2 k3 ndu ndf δ out2 ccall((:sb_vfe_create, LIB), Int32,
        (Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbNoise}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ref{SbNoise}, Ptr{Cvoid},
         Ref{Ptr{Cvoid}}, Ptr{Float64}, Ref{Int64}),
        ctx().h, uu, nu, xu, ffd, nf, δ, h, out2, info)
    check(st, info[])
    V = VfeHandle(h[]); finalizer(destroy!, V)
    V, out2[1], out2[2]
end

elbo(v::AbstractGPs.VFE{<:B200Finite}, fx::B200Finite, y::AbstractVector{<:Real}) = vfe_create(v.fz, fx, y)[2]
dtc(v::AbstractGPs.VFE{<:B200Finite}, fx::B200Finite, y::AbstractVector{<:Real}) = vfe_create(v.fz, fx, y)[3]
function posterior(v::AbstractGPs.VFE{<:B200Finite}, fx::B200Finite, y::AbstractVector{<:Real})
    B200ApproxPosteriorGP(fx.f, v.fz.x, vfe_create(v.fz, fx, y)[1])
end

# SparseFiniteGP(fobs, finducing): logpdf == elbo, posterior == VFE posterior (sparse_finite_gp.jl:52-62)
const B200Sparse = SparseFiniteGP{<:B200Finite,<:B200Finite}
elbo(f::B200Sparse, y::AbstractVector{<:Real}) = elbo(AbstractGPs.VFE(f.finducing), f.fobs, y)
logpdf(f::B200Sparse, y::AbstractVector{<:Real}) = elbo(AbstractGPs.VFE(f.finducing), f.fobs, y)
logpdf(f::B200Sparse, Y::AbstractMatrix{<:Real}) = map(y -> logpdf(f, y), eachcol(Y))
posterior(f::B200Sparse, y::AbstractVector{<:Real}) = posterior(AbstractGPs.VFE(f.finducing), f.fobs, y)

function mean_and_var(fp::B200ApproxPosteriorGP, xs::AbstractVector)
    ps, vs = components(fp.prior, xs); pz, vz = components(fp.prior, fp.z)
    cross, k1 = build_spec(ps, vs, pz, vz; which=:all)
    pd, k2 = build_spec(ps, vs, ps, vs; which=:diag)
    n = npoints(xs); m = zeros(n); v = zeros(n)
    GC.@preserve k1 k2 m v check(ccall((:sb_vfe_predict, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ptr{Cvoid}, Ptr{Cvoid}),
        ctx().h, fp.V.h, cross, pd, m, v))
    m .+ lowered_mean(fp.prior, xs), v
end
mean(fp::B200ApproxPosteriorGP, xs::AbstractVector) = mean_and_var(fp, xs)[1]
var(fp::B200ApproxPosteriorGP, xs::AbstractVector) = mean_and_var(fp, xs)[2]
function cov(fp::B200ApproxPosteriorGP, xs::AbstractVector)
    ps, vs = components(fp.prior, xs); pz, vz = components(fp.prior, fp.z)
    cross, k1 = build_spec(ps, vs, pz, vz; which=:all)
    full, k2 = build_spec(ps, vs, ps, vs; which=:all)
    n = npoints(xs); K = Matrix{Float64}(undef, n, n)
    GC.@preserve k1 k2 K check(ccall((:sb_vfe_predict_cov, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ptr{Cvoid}), ctx().h, fp.V.h, cross, full, K))
    K
end

# ---- gradients of logpdf (what Zygote + ChainRules deliver in the reference, cross.jl:8-22) -----------
# returns (g_terms, g_noise_diag): g_terms[2t-1] = d/d coeff_t, g_terms[2t] = d/d log(input scale_t) per
# term of the symmetric spec, g_noise_diag[i] = d/d Sigma_y[i,i]; the caller applies its chain rule.
function logpdf_grad(fx::B200Finite, y::AbstractVector{<:Real})
    fp = posterior(fx, y); install_alpha!(fp)
    ps, vs = components(fx.f, fx.x)
    spec, keep = build_spec(ps, vs, ps, vs; which=:sym)
    g = zeros(2 * max(1, Int(spec.nterms))); qd = zeros(npoints(fx.x))
    GC.@preserve keep g qd check(ccall((:sb_logpdf_grad, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ptr{Float64}, Ptr{Cvoid}), ctx().h, fp.F.h, spec, g, qd))
    g, qd
end

# ---- gradient of the elbo (reverse mode of elbo(VFE(fz), fx, y), sparse_finite_gp.jl:52-58) ---------------
# returns (elbo, g_uu, g_xu, g_ff, g_noise_u, g_noise_f): per term of cov(fz) / cov(f, x, z) / var(f, x) as in
# logpdf_grad, g_noise_u[i] = d/d (K_uu + jitter)[i,i], g_noise_f[i] = d/d Sigma_y[i,i].  The specs are built
# once and passed to both sb_vfe_create and sb_vfe_grad.
function elbo_grad(v::AbstractGPs.VFE{<:B200Finite}, fx::B200Finite, y::AbstractVector{<:Real})
    fz = v.fz
    fz.f === fx.f || throw(ArgumentError("VFE: inducing and observed FiniteGPs must share the prior"))
    length(y) == npoints(fx.x) || throw(DimensionMismatch("length(y) != length(fx)"))
    fx.Σy isa Diagonal || error("SthenoB200: VFE needs diagonal observation noise")
    pz, vz = components(fz.f, fz.x); px, vx = components(fx.f, fx.x)
    uu, k1 = build_spec(pz, vz, pz, vz; which=:sym)
    xu, k2 = build_spec(px, vx, pz, vz; which=:all)
    ffd, k3 = build_spec(px, vx, px, vx; which=:diag)
    nu, ndu = noise_struct(fz.Σy); nf, ndf = noise_struct(fx.Σy)
    δ = Float64.(y .- host_mean(fx))
    h = Ref{Ptr{Cvoid}}(C_NULL); out2 = zeros(2); info = Ref{Int64}(0)
    st = GC.@preserve k1 k2 k3 ndu ndf δ out2 ccall((:sb_vfe_create, LIB), Int32,
        (Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbNoise}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ref{SbNoise}, Ptr{Cvoid},
         Ref{Ptr{Cvoid}}, Ptr{Float64}, Ref{Int64}),
        ctx().h, uu, nu, xu, ffd, nf, δ, h, out2, info)
    check(st, info[])
    V = VfeHandle(h[]); finalizer(destroy!, V)
    guu = zeros(2 * max(1, Int(uu.nterms))); gxu = zeros(2 * max(1, Int(xu.nterms)))
    gff = zeros(2 * max(1, Int(ffd.nterms))); gnu = zeros(npoints(fz.x)); gnf = zeros(npoints(fx.x))
    GC.@preserve k1 k2 k3 ndf δ guu gxu gff gnu gnf check(ccall((:sb_vfe_grad, LIB), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ref{SbCovSpec}, Ref{SbNoise}, Ptr{Cvoid},
         Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Cvoid}, Ptr{Cvoid}),
        ctx().h, V.h, uu, xu, ffd, nf, δ, guu, gxu, gff, gnu, gnf))
    out2[1], guu, gxu, gff, gnu, gnf
end

# ---- factor checkpoint / resume --------------------------------------------------------------------------
function save_factor(F::Factor)
    n = Ref{Int64}(0)
    check(ccall((:sb_factor_export_size, LIB), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{Int64}), ctx().h, F.h, n))
    blob = Vector{UInt8}(undef, n[])
    GC.@preserve blob check(ccall((:sb_factor_export, LIB), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64),
                                  ctx().h, F.h, blob, n[]))
    blob
end
function load_factor(blob::Vector{UInt8}, n::Integer)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve blob check(ccall((:sb_factor_import, LIB), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ref{Ptr{Cvoid}}),
                                  ctx().h, blob, length(blob), h))
    F = Factor(h[], n, nothing); finalizer(destroy!, F); F
end

# ---- timings (CUDA-event phase timers of the library) ------------------------------------------------
struct SbTimings
    assemble_ms::Float64; panel_ms::Float64; trailing_ms::Float64; solve_ms::Float64; predict_ms::Float64
    comm_ms::Float64; total_ms::Float64; trailing_flops::Float64; trailing_kernel_ms::Float64
    trailing_launches::Int64; kernel_launches::Int64; trailing_int8_ops::Float64; panel_chain_ms::Float64
end
function timings(; reset::Bool=false)
    t = Ref{SbTimings}()
    check(ccall((:sb_ctx_timings, LIB), Int32, (Ptr{Cvoid}, Ref{SbTimings}, Int32), ctx().h, t, reset ? 1 : 0))
    t[]
end

# "trailing" => 0 (fp64 DMMA) | 1 (int8 Ozaki slices on wgmma); default 0
set_option!(key::AbstractString, value::Integer) =
    check(ccall((:sb_ctx_set_option, LIB), Int32, (Ptr{Cvoid}, Cstring, Int64), ctx().h, key, value))

export b200, B200GPPP, timings, set_option!, logpdf_grad, elbo_grad, save_factor, load_factor

end # module
