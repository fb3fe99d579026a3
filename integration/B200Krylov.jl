# B200Krylov.jl -- the reference-side binding of libb200krylov.so (INTEGRATION.md).
#
# SOURCE ONLY: Julia is not installed in the build image, so this file has never been executed there.  It
# is the file a maintainer of IterativeSolvers.jl would add (or ship as a package extension): device
# operator / vector types plus methods of the five solver entry points that dispatch on them.  Every ccall
# below is exercised, with the same argument meaning, by the Python harness (iterativesolvers.jl_b200/_lib.py,
# whose signature table tests/test_abi_and_host.py checks against include/b200krylov.h).
#
# Keyword names, defaults and return shapes are the reference's: src/cg.jl:209-217, src/chebyshev.jl:131-139,
# src/gmres.jl:184-194, src/minres.jl:200-207, src/bicgstabl.jl:181-188, src/lobpcg.jl:827-829, and for the
# SURVEY section 8(f) widening src/qmr.jl:262-272, src/lsqr.jl:66-69,90-94, src/lsmr.jl:67-70,88-92, src/idrs.jl:49-56.
module B200Krylov

using SparseArrays, LinearAlgebra
import IterativeSolvers
import IterativeSolvers: cg!, chebyshev!, gmres!, minres!, bicgstabl!, lobpcg, qmr!, lsqr!, lsmr!, idrs!, svdl, powm!, invpowm!,
                         ConvergenceHistory, Identity, ClassicalGramSchmidt, ModifiedGramSchmidt, DGKS,
                         OrthogonalizationMethod, LOBPCGResults
import LinearAlgebra: mul!, ldiv!

const LIB = "libb200krylov.so"

check(status::Integer) =
    status == 0 ? nothing : error(unsafe_string(ccall((:b200_last_error, LIB), Cstring, ())))

# ------------------------------------------------------------------------------------------- context
mutable struct Ctx
    h::Ptr{Cvoid}
    function Ctx(device::Integer = 0)
        r = Ref{Ptr{Cvoid}}()
        check(ccall((:b200_ctx_create, LIB), Cint, (Cint, Ref{Ptr{Cvoid}}), device, r))
        finalizer(c -> ccall((:b200_ctx_destroy, LIB), Cint, (Ptr{Cvoid},), c.h), new(r[]))
    end
end
const DEFAULT_CTX = Ref{Union{Nothing,Ctx}}(nothing)
default_ctx() = something(DEFAULT_CTX[], (DEFAULT_CTX[] = Ctx(0)))

dtype_code(::Type{Float64}) = Cint(0)
dtype_code(::Type{Float32}) = Cint(1)
dtype_code(::Type{ComplexF64}) = Cint(2)   # interleaved (re, im): Complex{T}'s own memory layout
dtype_code(::Type{ComplexF32}) = Cint(3)
const BlasReal = Union{Float32,Float64}
# element types of device vectors and operators; complex ones are served by mul!, the BLAS-1 calls, cg! and gmres!
# (the other entry points return B200_ERR_UNSUPPORTED for them)
const B200Eltype = Union{Float32,Float64,ComplexF32,ComplexF64}

# ------------------------------------------------------------------------------------------- vectors
mutable struct B200Vector{T<:B200Eltype} <: AbstractVector{T}
    p::Ptr{T}
    n::Int
    ctx::Ctx
    function B200Vector{T}(ctx::Ctx, n::Integer) where {T}
        r = Ref{Ptr{Cvoid}}()
        check(ccall((:b200_malloc, LIB), Cint, (Ptr{Cvoid}, Csize_t, Ref{Ptr{Cvoid}}), ctx.h, n * sizeof(T), r))
        finalizer(v -> ccall((:b200_free, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), v.ctx.h, v.p),
                  new{T}(Ptr{T}(r[]), n, ctx))
    end
    # non-owning view of device memory the library hands to an operator callback (no finalizer)
    B200Vector{T}(ctx::Ctx, p::Ptr{T}, n::Integer, owner::Bool) where {T} = new{T}(p, n, ctx)
end
Base.size(v::B200Vector) = (v.n,)
Base.similar(v::B200Vector{T}) where {T} = B200Vector{T}(v.ctx, v.n)
function B200Vector(ctx::Ctx, x::Vector{T}) where {T<:B200Eltype}
    v = B200Vector{T}(ctx, length(x))
    check(ccall((:b200_upload, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t), ctx.h, v.p, x, sizeof(x)))
    v
end
function Base.Array(v::B200Vector{T}) where {T}
    x = Vector{T}(undef, v.n)
    check(ccall((:b200_download, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t), v.ctx.h, x, v.p, sizeof(x)))
    x
end
# operator-level BLAS-1: lets the UNMODIFIED reference loops (src/cg.jl:43-66, src/minres.jl:97-159) run on
# device vectors, one ccall per Julia operation
LinearAlgebra.dot(x::B200Vector{T}, y::B200Vector{T}) where {T<:BlasReal} = (r = Ref{Cdouble}();
    check(ccall((:b200_dot, LIB), Cint, (Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ref{Cdouble}),
                x.ctx.h, x.n, x.p, y.p, dtype_code(T), r)); T(r[]))
# dot(x, y) = sum(conj(x) .* y) for complex vectors
LinearAlgebra.dot(x::B200Vector{T}, y::B200Vector{T}) where {T<:Union{ComplexF32,ComplexF64}} = (r = zeros(Cdouble, 2);
    check(ccall((:b200_dotc, LIB), Cint, (Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Cdouble}),
                x.ctx.h, x.n, x.p, y.p, dtype_code(T), r)); T(complex(r[1], r[2])))
LinearAlgebra.norm(x::B200Vector{T}) where {T} = (r = Ref{Cdouble}();
    check(ccall((:b200_nrm2, LIB), Cint, (Ptr{Cvoid}, Int64, Ptr{Cvoid}, Cint, Ref{Cdouble}),
                x.ctx.h, x.n, x.p, dtype_code(T), r)); real(T)(r[]))
# y = a*x + b*y
axpby!(a, x::B200Vector{T}, b, y::B200Vector{T}) where {T} =
    (check(ccall((:b200_axpby, LIB), Cint, (Ptr{Cvoid}, Int64, Cdouble, Ptr{Cvoid}, Cdouble, Ptr{Cvoid}, Cint),
                 x.ctx.h, x.n, a, x.p, b, y.p, dtype_code(T))); y)
LinearAlgebra.axpy!(a, x::B200Vector, y::B200Vector) = axpby!(a, x, 1, y)
LinearAlgebra.rmul!(x::B200Vector{T}, a::Number) where {T} =
    (check(ccall((:b200_scal, LIB), Cint, (Ptr{Cvoid}, Int64, Cdouble, Ptr{Cvoid}, Cint), x.ctx.h, x.n, a, x.p, dtype_code(T))); x)
Base.copyto!(y::B200Vector{T}, x::B200Vector{T}) where {T} =
    (check(ccall((:b200_copy, LIB), Cint, (Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Cint), x.ctx.h, x.n, x.p, y.p, dtype_code(T))); y)
Base.fill!(x::B200Vector{T}, a::Number) where {T} =
    (check(ccall((:b200_fill, LIB), Cint, (Ptr{Cvoid}, Int64, Cdouble, Ptr{Cvoid}, Cint), x.ctx.h, x.n, a, x.p, dtype_code(T))); x)

# ------------------------------------------------------------------------------------------- operator
mutable struct B200CSR{T<:B200Eltype}
    h::Ptr{Cvoid}
    ctx::Ctx
    n::Int                                  # size(A, 1)
    ncols::Int                              # size(A, 2)  (rectangular operators: lsqr!/lsmr!)
    adj::Union{Nothing,B200CSR{T}}          # adjoint(A), built on first use
end
# stands where a SparseMatrixCSC is passed today (src/cg.jl:54, src/gmres.jl:287, ...): CSC -> device CSR int32
function B200CSR(A::SparseMatrixCSC{T,Ti}; ctx::Ctx = default_ctx()) where {T<:B200Eltype,Ti<:Union{Int32,Int64}}
    r = Ref{Ptr{Cvoid}}()
    check(ccall((:b200_csr_from_csc, LIB), Cint,
                (Ptr{Cvoid}, Int64, Int64, Ptr{Ti}, Ptr{Ti}, Ptr{T}, Cint, Cint, Cint, Ref{Ptr{Cvoid}}),
                ctx.h, size(A, 1), size(A, 2), A.colptr, A.rowval, A.nzval, sizeof(Ti), dtype_code(T), 1, r))
    finalizer(a -> ccall((:b200_csr_destroy, LIB), Cint, (Ptr{Cvoid},), a.h),
              B200CSR{T}(r[], ctx, size(A, 1), size(A, 2), nothing))
end
Base.size(A::B200CSR) = (A.n, A.ncols)
Base.size(A::B200CSR, d::Integer) = d == 1 ? A.n : (d == 2 ? A.ncols : 1)
Base.eltype(::B200CSR{T}) where {T} = T
# adjoint(A) as a device operator of its own (what LanczosDecomp stores, src/qmr.jl:54; lsqr src/lsqr.jl:128)
function Base.adjoint(A::B200CSR{T}) where {T}
    if A.adj === nothing
        r = Ref{Ptr{Cvoid}}()
        check(ccall((:b200_csr_transpose, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{Ptr{Cvoid}}), A.ctx.h, A.h, r))
        A.adj = finalizer(a -> ccall((:b200_csr_destroy, LIB), Cint, (Ptr{Cvoid},), a.h),
                          B200CSR{T}(r[], A.ctx, A.ncols, A.n, nothing))
    end
    A.adj
end
mul!(y::B200Vector{T}, A::B200CSR{T}, x::B200Vector{T}) where {T} =
    (check(ccall((:b200_spmv, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), A.ctx.h, A.h, x.p, y.p)); y)
# the device operator back as a SparseMatrixCSC{T,Int64}: its CSR is the CSC of transpose(A) (no conjugation).  Row
# offsets come through b200_csr_download64, which serves 4-byte and 8-byte operators alike.
function SparseArrays.SparseMatrixCSC(A::B200CSR{T}) where {T}
    nnz = Ref{Int64}(0)
    check(ccall((:b200_csr_info, LIB), Cint, (Ptr{Cvoid}, Ptr{Int64}, Ptr{Int64}, Ref{Int64}, Ptr{Cint}, Ptr{Int64}, Ptr{Int64}),
                A.h, C_NULL, C_NULL, nnz, C_NULL, C_NULL, C_NULL))
    rowptr = Vector{Int64}(undef, A.n + 1)
    colind = Vector{Int32}(undef, nnz[])
    vals = Vector{T}(undef, nnz[])
    check(ccall((:b200_csr_download64, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Int64}, Ptr{Int32}, Ptr{T}),
                A.ctx.h, A.h, rowptr, colind, vals))
    transpose(SparseMatrixCSC(A.ncols, A.n, rowptr .+ 1, Int64.(colind) .+ 1, vals)) |> SparseMatrixCSC
end

# the diagonal preconditioner of test/cg.jl:14-18
struct JacobiPrec{T}
    d::B200Vector{T}
end
function JacobiPrec(A::B200CSR{T}) where {T}
    d = B200Vector{T}(A.ctx, A.n)
    check(ccall((:b200_csr_diag, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), A.ctx.h, A.h, d.p))
    JacobiPrec{T}(d)
end
ldiv!(y::B200Vector{T}, P::JacobiPrec{T}, x::B200Vector{T}) where {T} =
    (check(ccall((:b200_jacobi_ldiv, LIB), Cint, (Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint),
                 x.ctx.h, x.n, P.d.p, x.p, y.p, dtype_code(T))); y)
ldiv!(P::JacobiPrec, x::B200Vector) = ldiv!(x, P, x)

# ------------------------------------------------------------------------------------------- C structs
struct Precond
    kind::Int32
    reserved::Int32
    diag::Ptr{Cvoid}
end
prec(::Identity) = Precond(0, 0, C_NULL)
prec(P::JacobiPrec) = Precond(1, 0, P.d.p)
prec(P) = throw(ArgumentError("the device path supports Identity() and JacobiPrec; got $(typeof(P))"))

mutable struct Result
    iters::Int64
    mvps::Int64
    isconverged::Int32
    status::Int32
    tol::Float64
    residual::Float64
    n_resnorm::Int64
    Result() = new(0, 0, 0, 0, 0.0, 0.0, 0)
end
struct CgOpts
    abstol::Float64; reltol::Float64; maxiter::Int64; initially_zero::Int32; check_every::Int32
    Pl::Precond; fixed_iterations::Int32; variant::Int32
end
struct GmresOpts
    abstol::Float64; reltol::Float64; maxiter::Int64; restart::Int32; initially_zero::Int32
    orth_meth::Int32; reserved::Int32; Pl::Precond; Pr::Precond
end
struct MinresOpts
    abstol::Float64; reltol::Float64; maxiter::Int64; initially_zero::Int32; skew_hermitian::Int32
end
struct BicgstablOpts
    abstol::Float64; reltol::Float64; max_mv_products::Int64; l::Int32; initial_zero::Int32
    Pl::Precond; r_shadow::Ptr{Cvoid}
end
struct LobpcgOpts
    tol::Float64; maxiter::Int64; largest::Int32; blocksize::Int32; P::Precond
    fixed_iterations::Int32; reserved::Int32
    trace_resnorm::Ptr{Float64}; trace_ritz::Ptr{Float64}; trace_cap::Int64      # log = true: one row per iteration
end
mutable struct LobpcgResult
    iterations::Int64; converged::Int32; status::Int32
    LobpcgResult() = new(0, 0, 0)
end
struct QmrOpts
    abstol::Float64; reltol::Float64; maxiter::Int64; initially_zero::Int32; check_every::Int32
end
struct LsqOpts
    damp::Float64; atol::Float64; btol::Float64; conlim::Float64; maxiter::Int64; check_every::Int32; reserved::Int32
end
mutable struct LsqResult
    iters::Int64; mvps::Int64; mtvps::Int64; isconverged::Int32; istop::Int32; status::Int32; reserved::Int32
    n_hist::Int64; hist_stride::Int64; atol::Float64; btol::Float64; ctol::Float64
    LsqResult() = new(0, 0, 0, 0, 0, 0, 0, 0, 0, 0.0, 0.0, 0.0)
end
struct IdrsOpts
    abstol::Float64; reltol::Float64; maxiter::Int64; s::Int32; smoothing::Int32; Pl::Precond
    P::Ptr{Cvoid}; ldp::Int64; check_every::Int32; reserved::Int32
end
struct LinOp                                   # b200_linop
    apply::Ptr{Cvoid}; user::Ptr{Cvoid}; m_local::Int64; n_local::Int64; n_global::Int64; m_global::Int64
    dtype::Int32; reserved::Int32
end
orth_code(::ModifiedGramSchmidt) = Int32(0); orth_code(::ClassicalGramSchmidt) = Int32(1); orth_code(::DGKS) = Int32(2)   # B200_ORTH_*

function history(res::Result, resnorm, abstol, reltol; restart = nothing)
    h = ConvergenceHistory(partial = false, restart = restart)
    h[:abstol] = abstol; h[:reltol] = reltol; h[:tol] = res.tol
    h.mvps = res.mvps; h.iters = res.iters; h.isconverged = res.isconverged != 0
    h.data[:resnorm] = resnorm[1:res.n_resnorm]
    h
end

# host x, b: upload, solve on the device, download x into the caller's array (in place, src/cg.jl:241)
function staged(f, A::B200CSR{T}, x::Vector{T}, b::Vector{T}) where {T}
    xd, bd = B200Vector(A.ctx, x), B200Vector(A.ctx, b)
    f(xd, bd)
    copyto!(x, Array(xd))
    x
end

# ------------------------------------------------------------------------------------------- cg!
function cg!(x::B200Vector{T}, A::B200CSR{T}, b::B200Vector{T};
             abstol::Real = zero(real(T)), reltol::Real = sqrt(eps(real(T))), maxiter::Int = size(A, 2), log::Bool = false,
             verbose::Bool = false, Pl = Identity(), initially_zero::Bool = false, kwargs...) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter + 1 : 0)
    o = CgOpts(abstol, reltol, maxiter, initially_zero, 0, prec(Pl), 0, 0)
    check(ccall((:b200_cg_solve, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{CgOpts}, Ref{Result}, Ptr{Float64}, Int64),
                A.ctx.h, A.h, x.p, b.p, o, res, hist, length(hist)))
    log ? (x, history(res, hist, abstol, reltol)) : x
end
# host arrays: one call does H2D of b and x, the solve, D2H of x
function cg!(x::Vector{T}, A::B200CSR{T}, b::Vector{T};
             abstol::Real = zero(real(T)), reltol::Real = sqrt(eps(real(T))), maxiter::Int = size(A, 2), log::Bool = false,
             verbose::Bool = false, Pl = Identity(), initially_zero::Bool = false, kwargs...) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter + 1 : 0)
    o = CgOpts(abstol, reltol, maxiter, initially_zero, 0, prec(Pl), 0, 0)
    check(ccall((:b200_cg_solve_host, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{T}, Ptr{T}, Ref{CgOpts}, Ref{Result}, Ptr{Float64}, Int64),
                A.ctx.h, A.h, x, b, o, res, hist, length(hist)))
    log ? (x, history(res, hist, abstol, reltol)) : x
end

# cg_iterator! (src/cg.jl:120-155): `for (k, residual) in enumerate(it)` as in docs/src/iterators.md
mutable struct B200CGIterable{T}
    h::Ptr{Cvoid}
    x::B200Vector{T}
    res::Result
end
function IterativeSolvers.cg_iterator!(x::B200Vector{T}, A::B200CSR{T}, b::B200Vector{T}, Pl = Identity();
                                       abstol::Real = zero(T), reltol::Real = sqrt(eps(T)), maxiter::Int = size(A, 2),
                                       statevars = nothing, initially_zero::Bool = false) where {T}
    o = CgOpts(abstol, reltol, maxiter, initially_zero, 0, prec(Pl), 0, 0)
    r = Ref{Ptr{Cvoid}}()
    u, rr, c = statevars === nothing ? (C_NULL, C_NULL, C_NULL) : (statevars.u.p, statevars.r.p, statevars.c.p)
    check(ccall((:b200_cg_iter_create, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{CgOpts}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{Ptr{Cvoid}}),
                A.ctx.h, A.h, x.p, b.p, o, u, rr, c, r))
    it = B200CGIterable{T}(r[], x, Result())
    step!(it, 0)
    finalizer(i -> ccall((:b200_cg_iter_destroy, LIB), Cint, (Ptr{Cvoid},), i.h), it)
end
step!(it::B200CGIterable, k::Integer) =
    check(ccall((:b200_cg_iter_next, LIB), Cint, (Ptr{Cvoid}, Int64, Ref{Result}, Ptr{Float64}, Int64), it.h, k, it.res, C_NULL, 0))
function Base.iterate(it::B200CGIterable, iteration::Int = 0)
    it.res.status == 1 && return nothing                    # done(it, iteration)  src/cg.jl:36
    step!(it, 1)
    it.res.residual, iteration + 1                           # src/cg.jl:65
end

# ------------------------------------------------------------------------------------------- chebyshev!
function chebyshev!(x::Vector{T}, A::B200CSR{T}, b::Vector{T}, λmin::Real, λmax::Real;
                    abstol::Real = zero(T), reltol::Real = sqrt(eps(T)), Pl = Identity(), maxiter::Int = size(A, 2),
                    log::Bool = false, verbose::Bool = false, initially_zero::Bool = false) where {T}
    res = Result(); hist = Vector{Float64}(undef, maxiter)
    o = CgOpts(abstol, reltol, maxiter, initially_zero, 0, prec(Pl), 0, 0)
    staged(A, x, b) do xd, bd
        check(ccall((:b200_chebyshev_solve, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cdouble, Cdouble, Ref{CgOpts}, Ref{Result}, Ptr{Float64}, Int64),
                    A.ctx.h, A.h, xd.p, bd.p, λmin, λmax, o, res, hist, length(hist)))
    end
    log ? (x, history(res, hist, abstol, reltol)) : x
end

# ------------------------------------------------------------------------------------------- gmres!
function gmres!(x::Vector{T}, A::B200CSR{T}, b::Vector{T};
                Pl = Identity(), Pr = Identity(), abstol::Real = zero(real(T)), reltol::Real = sqrt(eps(real(T))),
                restart::Int = min(20, size(A, 2)), maxiter::Int = size(A, 2), log::Bool = false,
                initially_zero::Bool = false, verbose::Bool = false,
                orth_meth::OrthogonalizationMethod = ModifiedGramSchmidt()) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter : 0)
    o = GmresOpts(abstol, reltol, maxiter, restart, initially_zero, orth_code(orth_meth), 0, prec(Pl), prec(Pr))
    staged(A, x, b) do xd, bd
        check(ccall((:b200_gmres_solve, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{GmresOpts}, Ref{Result}, Ptr{Float64}, Int64),
                    A.ctx.h, A.h, xd.p, bd.p, o, res, hist, length(hist)))
    end
    log ? (x, history(res, hist, abstol, reltol; restart = restart)) : x
end

# ------------------------------------------------------------------------------------------- minres!
function minres!(x::Vector{T}, A::B200CSR{T}, b::Vector{T};
                 skew_hermitian::Bool = false, verbose::Bool = false, log::Bool = false, abstol::Real = zero(T),
                 reltol::Real = sqrt(eps(T)), maxiter::Int = size(A, 2), initially_zero::Bool = false) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter : 0)
    o = MinresOpts(abstol, reltol, maxiter, initially_zero, skew_hermitian)
    staged(A, x, b) do xd, bd
        check(ccall((:b200_minres_solve, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{MinresOpts}, Ref{Result}, Ptr{Float64}, Int64),
                    A.ctx.h, A.h, xd.p, bd.p, o, res, hist, length(hist)))
    end
    log ? (x, history(res, hist, abstol, reltol)) : x
end

# ------------------------------------------------------------------------------------------- bicgstabl!
function bicgstabl!(x::Vector{T}, A::B200CSR{T}, b::Vector{T}, l::Int = 2;
                    abstol::Real = zero(T), reltol::Real = sqrt(eps(T)), max_mv_products::Int = size(A, 2),
                    log::Bool = false, verbose::Bool = false, Pl = Identity(), initial_zero::Bool = false) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? max_mv_products : 0)
    shadow = B200Vector(A.ctx, rand(T, length(b)))            # r_shadow = rand(T, n)  src/bicgstabl.jl:38
    o = BicgstablOpts(abstol, reltol, max_mv_products, l, initial_zero, prec(Pl), shadow.p)
    GC.@preserve shadow staged(A, x, b) do xd, bd
        status = ccall((:b200_bicgstabl_solve, LIB), Cint,
                       (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{BicgstablOpts}, Ref{Result}, Ptr{Float64}, Int64),
                       A.ctx.h, A.h, xd.p, bd.p, o, res, hist, length(hist))
        status == -5 && throw(SingularException(0))           # lu! of the MR matrix, src/bicgstabl.jl:123
        check(status)
    end
    log ? (x, history(res, hist, abstol, reltol)) : x
end

# ------------------------------------------------------------------------------------------- lobpcg
function lobpcg(A::B200CSR{T}, largest::Bool, X0::Matrix{T}; P = nothing, tol::Real = eps(T)^(3 / 10),
                maxiter::Integer = 200, log::Bool = false) where {T}
    n, bs = size(X0)
    n == size(A, 1) || throw(DimensionMismatch("X0 has $n rows, A has $(size(A, 1))"))
    Xd = B200Vector(A.ctx, vec(copy(X0)))                     # X0 is copied  src/lobpcg.jl:830
    λ = Vector{Float64}(undef, bs); rn = Vector{Float64}(undef, bs)
    res = LobpcgResult()
    tr_r = log ? Matrix{Float64}(undef, bs, maxiter) : Matrix{Float64}(undef, 0, 0)     # LOBPCGState per iteration :744-745
    tr_l = log ? Matrix{Float64}(undef, bs, maxiter) : Matrix{Float64}(undef, 0, 0)
    o = LobpcgOpts(tol, maxiter, largest, bs, P === nothing ? prec(Identity()) : prec(P), 0, 0,
                   log ? pointer(tr_r) : C_NULL, log ? pointer(tr_l) : C_NULL, log ? maxiter : 0)
    status = GC.@preserve tr_r tr_l ccall((:b200_lobpcg_solve, LIB), Cint,
                   (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ref{LobpcgOpts}, Ref{LobpcgResult}, Ptr{Float64}, Ptr{Float64}),
                   A.ctx.h, A.h, Xd.p, n, o, res, λ, rn)
    status == -5 && throw(PosDefException(0))                 # cholesky! in CholQR  src/lobpcg.jl:380
    check(status)
    X = reshape(Array(Xd), n, bs)
    trace = log ? [LOBPCGState(i, T.(tr_r[:, i]), T.(tr_l[:, i])) for i in 1:min(Int(res.iterations), maxiter)] : nothing
    LOBPCGResults(T.(λ), X, T(tol), T.(rn), Int(res.iterations), Int(maxiter), res.converged != 0, trace)
end

# ------------------------------------------------------------------------------------------- qmr!  (SURVEY 8f item 4)
function qmr!(x::Vector{T}, A::B200CSR{T}, b::Vector{T};
              abstol::Real = zero(T), reltol::Real = sqrt(eps(T)), maxiter::Int = size(A, 2), lookahead::Bool = false,
              log::Bool = false, initially_zero::Bool = false, verbose::Bool = false) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter : 0)
    o = QmrOpts(abstol, reltol, maxiter, initially_zero, 0)
    At = adjoint(A)
    staged(A, x, b) do xd, bd
        check(ccall((:b200_qmr_solve, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{QmrOpts}, Ref{Result}, Ptr{Float64}, Int64),
                    A.ctx.h, A.h, At.h, xd.p, bd.p, o, res, hist, length(hist)))
    end
    if log
        h = history(res, hist, abstol, reltol)
        h.mvps = 0                                            # nextiter!(history) without mvps, src/qmr.jl:285
        return x, h
    end
    x
end

# ------------------------------------------------------------------------------------------- lsqr! / lsmr!
function ls_history(res::LsqResult, hist::Vector{Float64}, first::Union{Nothing,Symbol})
    h = ConvergenceHistory(partial = false)
    h[:atol] = res.atol; h[:btol] = res.btol; h[:ctol] = res.ctol
    h.mvps = res.mvps; h.mtvps = res.mtvps; h.iters = res.iters; h.isconverged = res.isconverged != 0
    sd = res.hist_stride; k = res.n_hist
    first === nothing || (h.data[first] = hist[1:k])
    h.data[:anorm] = hist[sd+1:sd+k]; h.data[:rnorm] = hist[2sd+1:2sd+k]; h.data[:cnorm] = hist[3sd+1:3sd+k]
    h
end
function ls_solve(sym::Symbol, first, x::Vector{T}, A::B200CSR{T}, b::Vector{T}, o::LsqOpts, maxiter::Int, log::Bool) where {T}
    length(x) == size(A, 2) || error("x should be of length ", size(A, 2))     # src/lsqr.jl:99
    length(b) == size(A, 1) || error("b should be of length ", size(A, 1))     # src/lsqr.jl:100
    res = LsqResult(); hist = Vector{Float64}(undef, 4 * max(maxiter, 1))
    At = adjoint(A)
    xd, bd = B200Vector(A.ctx, x), B200Vector(A.ctx, b)
    status = sym === :lsqr ?
        ccall((:b200_lsqr_solve, LIB), Cint,
              (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{LsqOpts}, Ref{LsqResult}, Ptr{Float64}, Int64),
              A.ctx.h, A.h, At.h, xd.p, bd.p, o, res, hist, maxiter) :
        ccall((:b200_lsmr_solve, LIB), Cint,
              (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{LsqOpts}, Ref{LsqResult}, Ptr{Float64}, Int64),
              A.ctx.h, A.h, At.h, xd.p, bd.p, o, res, hist, maxiter)
    status == -1 && res.status == -1 && error("Initial guess for x must be finite")   # src/lsqr.jl:102-104
    check(status)
    copyto!(x, Array(xd))
    log ? (x, ls_history(res, hist, first)) : x
end
function lsqr!(x::Vector{T}, A::B200CSR{T}, b::Vector{T};
               maxiter::Int = maximum(size(A)), log::Bool = false, damp = 0, atol = sqrt(eps(T)), btol = sqrt(eps(T)),
               conlim = one(T) / sqrt(eps(T)), verbose::Bool = false) where {T}
    ls_solve(:lsqr, :resnorm, x, A, b, LsqOpts(damp, atol, btol, conlim, maxiter, 0, 0), maxiter, log)
end
function lsmr!(x::Vector{T}, A::B200CSR{T}, b::Vector{T};
               maxiter::Int = maximum(size(A)), log::Bool = false, atol::Number = 1e-6, btol::Number = 1e-6,
               conlim::Number = 1e8, λ::Number = 0, verbose::Bool = false) where {T}
    ls_solve(:lsmr, nothing, x, A, b, LsqOpts(λ, atol, btol, conlim, maxiter, 0, 0), maxiter, log)
end

# ------------------------------------------------------------------------------------------- idrs!
function idrs!(x::Vector{T}, A::B200CSR{T}, b::Vector{T};
               s = 8, Pl = Identity(), abstol::Real = zero(T), reltol::Real = sqrt(eps(T)), maxiter = size(A, 2),
               log::Bool = false, smoothing::Bool = false, verbose::Bool = false) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter : 0)
    n = length(b)
    P = B200Vector(A.ctx, rand(T, n * s))                     # P = [rand!(copy(C)) for k in 1:s]  src/idrs.jl:132
    o = IdrsOpts(abstol, reltol, maxiter, s, smoothing, prec(Pl), P.p, n, 0, 0)
    GC.@preserve P staged(A, x, b) do xd, bd
        check(ccall((:b200_idrs_solve, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{IdrsOpts}, Ref{Result}, Ptr{Float64}, Int64),
                    A.ctx.h, A.h, xd.p, bd.p, o, res, hist, length(hist)))
    end
    log ? (x, history(res, hist, abstol, reltol)) : x
end

# ------------------------------------------------------------------------------------------- lobpcg: constraint, nev driver
mutable struct B200Constraint{T}                     # Constraint(Y, nothing, X)  src/lobpcg.jl:144-224 (B = I)
    h::Ptr{Cvoid}
    ctx::Ctx
end
function B200Constraint(A::B200CSR{T}, Y::Matrix{T}; capacity::Integer = size(Y, 2)) where {T}
    Yd = B200Vector(A.ctx, vec(Y)); r = Ref{Ptr{Cvoid}}()
    check(ccall((:b200_lobpcg_constraint_create, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Cvoid}, Int64, Cint, Cint, Cint, Ref{Ptr{Cvoid}}),
                A.ctx.h, size(Y, 1), Yd.p, size(Y, 1), size(Y, 2), capacity, dtype_code(T), r))
    finalizer(c -> ccall((:b200_lobpcg_constraint_destroy, LIB), Cint, (Ptr{Cvoid},), c.h), B200Constraint{T}(r[], A.ctx))
end
# update!(constr!, X[:, 1:k], ...)  src/lobpcg.jl:188-206
update!(c::B200Constraint, Xd::B200Vector, n::Integer, k::Integer) =
    check(ccall((:b200_lobpcg_constraint_append, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Cint),
                c.ctx.h, c.h, Xd.p, n, k))
# lobpcg(A, largest, X0; C = Y, ...): as `lobpcg` above with
#   ccall((:b200_lobpcg_solve_constrained, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ref{LobpcgOpts},
#         Ptr{Cvoid}, Ref{LobpcgResult}, Ptr{Float64}, Ptr{Float64}), A.ctx.h, A.h, Xd.p, n, o, c.h, res, λ, rn)
# lobpcg(A, largest, X0, nev; ...) (src/lobpcg.jl:925-962) is the same host loop as iterativesolvers.jl_b200/solvers.py:
# solve a block, update!(constraint, converged columns), rand! the block, repeat.

# ------------------------------------------------------------------------------------------- lobpcg(A, B, largest, X0)
# The generalized problem A x = λ B x (src/lobpcg.jl:824-839 with B given; LOBPCGIterator{true} :292-316), callback
# operators (B200LinearOperator: `mul!(y, A, x)`), a callback preconditioner, and a constraint in the B inner product
# (Constraint(Y, B, X) :162-186) go through the general engine.  b200_csr_as_linop wraps a CSR handle as a b200_linop
# whose `apply` is the library's own SpMV, so nothing crosses into Julia inside the iteration for CSR operands.
function as_linop(A::B200CSR{T}) where {T}
    r = Ref{LinOp}()
    check(ccall((:b200_csr_as_linop, LIB), Cint, (Ptr{Cvoid}, Ref{LinOp}), A.h, r)); r[]
end
function B200Constraint(A::B200CSR{T}, B::B200CSR{T}, Y::Matrix{T}; capacity::Integer = size(Y, 2)) where {T}   # Constraint(Y, B, X) :162-186
    Yd = B200Vector(A.ctx, vec(Y)); r = Ref{Ptr{Cvoid}}(); b = as_linop(B)
    check(ccall((:b200_lobpcg_constraint_create_b, LIB), Cint,
                (Ptr{Cvoid}, Ref{LinOp}, Int64, Ptr{Cvoid}, Int64, Cint, Cint, Cint, Ref{Ptr{Cvoid}}),
                A.ctx.h, b, size(Y, 1), Yd.p, size(Y, 1), size(Y, 2), capacity, dtype_code(T), r))
    finalizer(c -> ccall((:b200_lobpcg_constraint_destroy, LIB), Cint, (Ptr{Cvoid},), c.h), B200Constraint{T}(r[], A.ctx))
end
function lobpcg(A::B200CSR{T}, B::B200CSR{T}, largest::Bool, X0::Matrix{T}; P = nothing, C = nothing,
                tol::Real = eps(T)^(3 / 10), maxiter::Integer = 200, log::Bool = false) where {T}
    n, bs = size(X0)
    Xd = B200Vector(A.ctx, vec(copy(X0)))
    λ = Vector{Float64}(undef, bs); rn = Vector{Float64}(undef, bs); res = LobpcgResult()
    o = LobpcgOpts(tol, maxiter, largest, bs, P === nothing ? prec(Identity()) : prec(P), 0, 0, C_NULL, C_NULL, 0)
    con = C === nothing ? C_NULL : B200Constraint(A, B, C).h
    a = as_linop(A); b = as_linop(B)
    status = ccall((:b200_lobpcg_solve_op, LIB), Cint,
                   (Ptr{Cvoid}, Ref{LinOp}, Ref{LinOp}, Ptr{Cvoid}, Int64, Ref{LobpcgOpts}, Ptr{Cvoid}, Ref{LobpcgResult},
                    Ptr{Float64}, Ptr{Float64}), A.ctx.h, a, b, Xd.p, n, o, con, res, λ, rn)
    status == -5 && throw(PosDefException(0))                 # cholesky! in CholQR :380 / in the Rayleigh-Ritz step :455
    check(status)
    LOBPCGResults(T.(λ), reshape(Array(Xd), n, bs), T(tol), T.(rn), Int(res.iterations), Int(maxiter), res.converged != 0, nothing)
end

# ------------------------------------------------------------------------------------------- svdl
struct SvdlOpts
    nsv::Int32; k::Int32; j::Int32; method::Int32; maxiter::Int64; tol::Float64; reltol::Float64
    dolock::Int32; reserved::Int32
end
mutable struct SvdlResult
    iters::Int64; mvps::Int64; mtvps::Int64; isconverged::Int32; k::Int32; beta::Float64; tol::Float64
    SvdlResult() = new(0, 0, 0, 0, 0, 0.0, 0.0)
end
# svdl(A; nsv, k, tol, maxiter, method = :ritz, v0, j, reltol, vecs, dolock)  src/svdl.jl:157-247
function svdl(A::B200CSR{T}; nsv::Int = 6, k::Int = 2nsv, tol::Real = √eps(), maxiter::Int = minimum(size(A)),
                               method::Symbol = :ritz, log::Bool = false, j::Int = nsv, reltol::Real = √eps(),
                               v0::Vector{T} = (x = randn(T, size(A, 2)); x ./ norm(x)), vecs::Symbol = :none,
                               dolock::Bool = false) where {T}
    method in (:ritz, :harmonic) || throw(ArgumentError("Unknown restart method $method"))     # src/svdl.jl:193-200
    m, n = size(A); At = adjoint(A)
    v0d = B200Vector(A.ctx, v0); res = SvdlResult(); σ = Vector{Float64}(undef, nsv)
    Ud = vecs in (:left, :both) ? B200Vector{T}(A.ctx, m * nsv) : nothing
    Vd = vecs in (:right, :both) ? B200Vector{T}(A.ctx, n * nsv) : nothing
    ritz = zeros(k, maxiter); resn = zeros(nsv, maxiter); conv = zeros(Int32, nsv, maxiter); betas = zeros(maxiter); B = zeros(k, k)
    o = SvdlOpts(nsv, k, j, method == :harmonic ? 1 : 0, maxiter, tol, reltol, dolock, 0)
    check(ccall((:b200_svdl, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{SvdlOpts}, Ref{SvdlResult}, Ptr{Float64}, Ptr{Cvoid}, Int64,
                 Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}),
                A.ctx.h, A.h, At.h, v0d.p, o, res, σ, Ud === nothing ? C_NULL : Ud.p, m, Vd === nothing ? C_NULL : Vd.p, n,
                ritz, resn, conv, betas, B))
    values = T.(σ)
    X = vecs == :none ? values :
        LinearAlgebra.SVD(Ud === nothing ? zeros(T, m, 0) : reshape(Array(Ud), m, nsv), values,
                          Vd === nothing ? zeros(T, 0, n) : Matrix(reshape(Array(Vd), n, nsv)'))
    L = (B = B, β = res.beta)                              # the projected factorisation (P, Q stay on the device)
    log || return X, L
    h = ConvergenceHistory(partial = false); h[:tol] = res.tol
    h.iters = res.iters; h.mvps = res.mvps; h.mtvps = res.mtvps; h.isconverged = res.isconverged != 0
    it = res.iters
    h.data[:ritz] = ritz[:, 1:it]; h.data[:resnorm] = resn[:, 1:it]; h.data[:conv] = conv[:, 1:it] .!= 0; h.data[:betas] = betas[1:it]
    X, L, h
end

# ------------------------------------------------------------------------------------------- matrix-free operators
# Anything with mul!(y::B200Vector, A, x::B200Vector) (a LinearMap over device vectors, a user type, a closure) can be
# handed to the fused engines: the C library calls back between two of its kernels (b200_linop), on its own stream.
struct B200LinearOperator{T,F}
    f::F                                       # f(y::B200Vector{T}, x::B200Vector{T}) enqueues y = A x
    ctx::Ctx
    m::Int
    n::Int
end
function linop_thunk(user::Ptr{Cvoid}, x::Ptr{Cvoid}, y::Ptr{Cvoid}, stream::Ptr{Cvoid})::Cint
    op = unsafe_pointer_to_objref(user)::B200LinearOperator
    T = typeof(op).parameters[1]
    try
        op.f(B200Vector{T}(op.ctx, Ptr{T}(y), op.m, false), B200Vector{T}(op.ctx, Ptr{T}(x), op.n, false))   # non-owning views
        return Cint(0)
    catch
        return Cint(1)
    end
end
linop(op::B200LinearOperator{T}) where {T} =
    LinOp(@cfunction(linop_thunk, Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid})), pointer_from_objref(op),
          op.m, op.n, op.n, op.m, dtype_code(T), 0)

function cg!(x::B200Vector{T}, A::B200LinearOperator{T}, b::B200Vector{T};
             abstol::Real = zero(real(T)), reltol::Real = sqrt(eps(real(T))), maxiter::Int = A.n, log::Bool = false,
             Pl = Identity(), initially_zero::Bool = false, verbose::Bool = false) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter + 1 : 0)
    cb = Pl isa B200LinearOperator                                         # ldiv!(c, Pl, r) by callback
    o = CgOpts(abstol, reltol, maxiter, initially_zero, 0, cb ? prec(Identity()) : prec(Pl), 0, 0)
    a = Ref(linop(A)); p = cb ? Ref(linop(Pl)) : C_NULL
    GC.@preserve A Pl check(ccall((:b200_cg_solve_op, LIB), Cint,
        (Ptr{Cvoid}, Ptr{LinOp}, Ptr{LinOp}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{CgOpts}, Ref{Result}, Ptr{Float64}, Int64),
        A.ctx.h, a, p, x.p, b.p, o, res, hist, length(hist)))
    log ? (x, history(res, hist, abstol, reltol)) : x
end
# qmr!/lsqr!/lsmr!/idrs! on B200LinearOperator: the same pattern with b200_qmr_solve_op / b200_lsqr_solve_op /
# b200_lsmr_solve_op / b200_idrs_solve_op (the adjoint is a second B200LinearOperator).

# chebyshev!(x, A, b, λmin, λmax; Pl, ...) on a B200LinearOperator: as cg! above with
#   ccall((:b200_chebyshev_solve_op, LIB), Cint, (Ptr{Cvoid}, Ptr{LinOp}, Ptr{Cvoid}, Ptr{Cvoid}, Float64, Float64,
#         Ref{CgOpts}, Ref{Result}, Ptr{Float64}, Int64), A.ctx.h, a, x.p, b.p, λmin, λmax, o, res, hist, length(hist))
# and the preconditioner in o.Pl (prec_cb below).

# A preconditioner given as a B200LinearOperator (f(y, x) enqueues y = P \ x, i.e. ldiv!(y, P, x)) travels in the
# b200_precond slot as B200_PREC_CALLBACK = 2 with the address of its b200_linop; the Ref must outlive the call.
prec_cb(P, keep::Vector{Any}) = prec(P)
function prec_cb(P::B200LinearOperator, keep::Vector{Any})
    r = Ref(linop(P)); push!(keep, r)
    Precond(2, 0, Base.unsafe_convert(Ptr{Cvoid}, r))
end

# ------------------------------------------------------------------------------------------- ILU(0)
# Zero-fill incomplete LU factored on the device (b200_ilu0_*; what IncompleteLU.jl's ilu(A, τ = 0) would give on A's
# pattern, docs/src/preconditioning.md).  Float64 / Float32 operators; the factor reuses A's index arrays, so it keeps A.
# As Pl / Pr it travels as B200_PREC_CALLBACK with the library's own thunk (b200_ilu0_as_linop): no Julia in the loop.
mutable struct B200ILU0{T}
    h::Ptr{Cvoid}
    A::B200CSR{T}
end
function B200ILU0(A::B200CSR{T}) where {T<:Union{Float64,Float32}}
    r = Ref{Ptr{Cvoid}}()
    check(ccall((:b200_ilu0_create, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{Ptr{Cvoid}}), A.ctx.h, A.h, r))
    P = B200ILU0{T}(r[], A)
    finalizer(P -> ccall((:b200_ilu0_destroy, LIB), Cint, (Ptr{Cvoid},), P.h), P)
end
ldiv!(y::B200Vector{T}, P::B200ILU0{T}, x::B200Vector{T}) where {T} =
    (check(ccall((:b200_ilu0_ldiv, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), P.A.ctx.h, P.h, x.p, y.p)); y)
ldiv!(P::B200ILU0, x::B200Vector) = ldiv!(x, P, x)                 # in place: the solves allow x == y
Base.:\(P::B200ILU0{T}, x::B200Vector{T}) where {T} = ldiv!(B200Vector{T}(P.A.ctx, P.A.n), P, x)
function prec_cb(P::B200ILU0, keep::Vector{Any})
    r = Ref{LinOp}()
    check(ccall((:b200_ilu0_as_linop, LIB), Cint, (Ptr{Cvoid}, Ref{LinOp}), P.h, r)); push!(keep, r, P)
    Precond(2, 0, Base.unsafe_convert(Ptr{Cvoid}, r))
end

# ------------------------------------------------------------------------------------------- smoothed-aggregation AMG
# AlgebraicMultigrid.jl's aspreconditioner(smoothed_aggregation(A; θ, max_levels, max_coarse)) with weighted-Jacobi
# sweeps (b200_amg_*, DESIGN section 23): the hierarchy is built on the host, the V-cycle runs on the device.  Level 0 is
# A itself, so the preconditioner keeps A.  As Pl / Pr it travels as B200_PREC_CALLBACK with the library's own thunk.
struct AmgOpts
    theta::Float64
    max_levels::Int32
    max_coarse::Int32
    presweeps::Int32
    postsweeps::Int32
end
mutable struct B200SmoothedAggregation{T}
    h::Ptr{Cvoid}
    A::B200CSR{T}
end
function B200SmoothedAggregation(A::B200CSR{T}; θ::Real = 0.0, max_levels::Integer = 10, max_coarse::Integer = 10,
                                 presweeps::Integer = 1, postsweeps::Integer = 1) where {T<:Union{Float64,Float32}}
    r = Ref{Ptr{Cvoid}}()
    o = Ref(AmgOpts(θ, max_levels, max_coarse, presweeps, postsweeps))
    check(ccall((:b200_amg_create, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{AmgOpts}, Ref{Ptr{Cvoid}}), A.ctx.h, A.h, o, r))
    P = B200SmoothedAggregation{T}(r[], A)
    finalizer(P -> ccall((:b200_amg_destroy, LIB), Cint, (Ptr{Cvoid},), P.h), P)
end
ldiv!(y::B200Vector{T}, P::B200SmoothedAggregation{T}, x::B200Vector{T}) where {T} =
    (check(ccall((:b200_amg_ldiv, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), P.A.ctx.h, P.h, x.p, y.p)); y)
ldiv!(P::B200SmoothedAggregation, x::B200Vector) = ldiv!(x, P, x)    # in place: the V-cycle allows x == y
Base.:\(P::B200SmoothedAggregation{T}, x::B200Vector{T}) where {T} = ldiv!(B200Vector{T}(P.A.ctx, P.A.n), P, x)
function prec_cb(P::B200SmoothedAggregation, keep::Vector{Any})
    r = Ref{LinOp}()
    check(ccall((:b200_amg_as_linop, LIB), Cint, (Ptr{Cvoid}, Ref{LinOp}), P.h, r)); push!(keep, r, P)
    Precond(2, 0, Base.unsafe_convert(Ptr{Cvoid}, r))
end

# gmres!(x, A, b; Pl, Pr, ...) with `mul!` / `ldiv!` callbacks  src/gmres.jl:184-194 (expand! :285-304)
function gmres!(x::B200Vector{T}, A::Union{B200CSR{T},B200LinearOperator{T}}, b::B200Vector{T};
                Pl = Identity(), Pr = Identity(), abstol::Real = zero(real(T)), reltol::Real = sqrt(eps(real(T))),
                restart::Int = min(20, size(A, 2)), maxiter::Int = size(A, 2), log::Bool = false,
                initially_zero::Bool = false, verbose::Bool = false,
                orth_meth::OrthogonalizationMethod = ModifiedGramSchmidt()) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter : 0); keep = Any[]
    o = GmresOpts(abstol, reltol, maxiter, restart, initially_zero, orth_code(orth_meth), 0, prec_cb(Pl, keep), prec_cb(Pr, keep))
    GC.@preserve A Pl Pr keep begin
        if A isa B200LinearOperator
            a = Ref(linop(A))
            check(ccall((:b200_gmres_solve_op, LIB), Cint,
                        (Ptr{Cvoid}, Ptr{LinOp}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{GmresOpts}, Ref{Result}, Ptr{Float64}, Int64),
                        A.ctx.h, a, x.p, b.p, o, res, hist, length(hist)))
        else                                    # CSR operator: b200_gmres_solve forwards callback preconditioners
            check(ccall((:b200_gmres_solve, LIB), Cint,
                        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{GmresOpts}, Ref{Result}, Ptr{Float64}, Int64),
                        A.ctx.h, A.h, x.p, b.p, o, res, hist, length(hist)))
        end
    end
    log ? (x, history(res, hist, abstol, reltol; restart = restart)) : x
end

# minres!(x, A, b; ...) with a `mul!` callback  src/minres.jl:200-207
function minres!(x::B200Vector{T}, A::B200LinearOperator{T}, b::B200Vector{T};
                 skew_hermitian::Bool = false, verbose::Bool = false, log::Bool = false, abstol::Real = zero(T),
                 reltol::Real = sqrt(eps(T)), maxiter::Int = A.n, initially_zero::Bool = false) where {T}
    res = Result(); hist = Vector{Float64}(undef, log ? maxiter : 0)
    o = MinresOpts(abstol, reltol, maxiter, initially_zero, skew_hermitian); a = Ref(linop(A))
    GC.@preserve A check(ccall((:b200_minres_solve_op, LIB), Cint,
        (Ptr{Cvoid}, Ptr{LinOp}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{MinresOpts}, Ref{Result}, Ptr{Float64}, Int64),
        A.ctx.h, a, x.p, b.p, o, res, hist, length(hist)))
    log ? (x, history(res, hist, abstol, reltol)) : x
end

# bicgstabl!(x, A, b, l; Pl, ...) with `mul!` / `ldiv!` callbacks  src/bicgstabl.jl:181-188
function bicgstabl!(x::B200Vector{T}, A::Union{B200CSR{T},B200LinearOperator{T}}, b::B200Vector{T}, l::Int = 2;
                    abstol::Real = zero(T), reltol::Real = sqrt(eps(T)), max_mv_products::Int = size(A, 2),
                    log::Bool = false, verbose::Bool = false, Pl = Identity(), initial_zero::Bool = false,
                    r_shadow::B200Vector{T} = B200Vector(A.ctx, rand(T, size(A, 1)))) where {T}      # rand(T, n) :38
    res = Result(); hist = Vector{Float64}(undef, log ? max_mv_products : 0); keep = Any[]
    o = BicgstablOpts(abstol, reltol, max_mv_products, l, initial_zero, prec_cb(Pl, keep), r_shadow.p)
    status = GC.@preserve A Pl keep r_shadow begin
        if A isa B200LinearOperator
            a = Ref(linop(A))
            ccall((:b200_bicgstabl_solve_op, LIB), Cint,
                  (Ptr{Cvoid}, Ptr{LinOp}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{BicgstablOpts}, Ref{Result}, Ptr{Float64}, Int64),
                  A.ctx.h, a, x.p, b.p, o, res, hist, length(hist))
        else
            ccall((:b200_bicgstabl_solve, LIB), Cint,
                  (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{BicgstablOpts}, Ref{Result}, Ptr{Float64}, Int64),
                  A.ctx.h, A.h, x.p, b.p, o, res, hist, length(hist))
        end
    end
    status == -5 && throw(SingularException(0))                            # lu! in the MR step  src/bicgstabl.jl:123
    check(status)
    log ? (x, history(res, hist, abstol, reltol)) : x
end
# gmres_iterable! / minres_iterable! / bicgstabl_iterator! (docs/src/iterators.md): b200_*_iter_create + b200_iter_next.
# `for (iteration, residual) in enumerate(it)` works as with the reference's iterables; x is updated in place.
mutable struct B200Iterable{T}
    h::Ptr{Cvoid}; ctx::Ctx; res::Result; x::B200Vector{T}; keep::Vector{Any}
end
function iter_finalize(it::B200Iterable)
    it.h == C_NULL || ccall((:b200_iter_destroy, LIB), Cint, (Ptr{Cvoid},), it.h); it.h = C_NULL
end
function gmres_iterable!(x::B200Vector{T}, A::Union{B200CSR{T},B200LinearOperator{T}}, b::B200Vector{T};
                         Pl = Identity(), Pr = Identity(), abstol::Real = zero(T), reltol::Real = sqrt(eps(T)),
                         restart::Int = min(20, size(A, 2)), maxiter::Int = size(A, 2), initially_zero::Bool = false,
                         orth_meth::OrthogonalizationMethod = ModifiedGramSchmidt()) where {T}
    keep = Any[A, Pl, Pr, b]; r = Ref{Ptr{Cvoid}}()
    o = GmresOpts(abstol, reltol, maxiter, restart, initially_zero, orth_code(orth_meth), 0, prec_cb(Pl, keep), prec_cb(Pr, keep))
    csr = A isa B200CSR ? A.h : C_NULL
    a = A isa B200LinearOperator ? (ar = Ref(linop(A)); push!(keep, ar); Base.unsafe_convert(Ptr{LinOp}, ar)) : Ptr{LinOp}(C_NULL)
    check(ccall((:b200_gmres_iter_create, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{LinOp}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{GmresOpts}, Ref{Ptr{Cvoid}}),
                A.ctx.h, csr, a, x.p, b.p, o, r))
    finalizer(iter_finalize, B200Iterable{T}(r[], A.ctx, Result(), x, keep))
end
# cg_iterator!(x, A::B200LinearOperator, b, Pl; ...): b200_cg_iter_create_op with Ref{CgOpts} (the CSR + Identity / Jacobi form
# with CGStateVariables is b200_cg_iter_create).
# minres_iterable!(x, A, b; ...) and bicgstabl_iterator!(x, A, b, l; ...): same pattern with b200_minres_iter_create
# (Ref{MinresOpts}) / b200_bicgstabl_iter_create (Ref{BicgstablOpts}).
function step!(it::B200Iterable, k::Integer = 1)
    buf = Vector{Float64}(undef, min(k, 4096))
    status = GC.@preserve it ccall((:b200_iter_next, LIB), Cint, (Ptr{Cvoid}, Int64, Ref{Result}, Ptr{Float64}, Int64),
                                   it.h, k, it.res, buf, length(buf))
    status == -5 && throw(SingularException(0)); check(status)
    resize!(buf, it.res.n_resnorm)
end
Base.iterate(it::B200Iterable, state = nothing) =
    it.res.status == 1 ? nothing : (r = step!(it, 1); isempty(r) ? nothing : (r[1], nothing))   # yields the residual norm
converged(it::B200Iterable) = it.res.isconverged != 0

# ------------------------------------------------------------------------------------------- powm! / invpowm!
struct PowmOpts
    tol::Float64; maxiter::Int64; shift::Float64; inverse::Int32; check_every::Int32
end
# powm!(B, x; shift, inverse, tol, maxiter, log)  src/simple.jl:118-151 ; invpowm!(B, x; ...) = powm!(...; inverse = true) :186
function powm!(B::Union{B200CSR{T},B200LinearOperator{T}}, x::B200Vector{T}; tol::Real = eps(T) * size(B, 2)^3,
               maxiter::Int = size(B, 1), shift::Real = zero(T), inverse::Bool = false, log::Bool = false,
               verbose::Bool = false) where {T}
    res = Result(); λ = Ref{Float64}(); hist = Vector{Float64}(undef, log ? maxiter + 1 : 0)
    o = PowmOpts(tol, maxiter, shift, inverse, 0)
    csr = B isa B200CSR ? B.h : C_NULL
    GC.@preserve B begin
        a = B isa B200LinearOperator ? Ref(linop(B)) : Ptr{LinOp}(C_NULL)
        check(ccall((:b200_powm, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{LinOp}, Ptr{Cvoid}, Ref{PowmOpts}, Ref{Result}, Ref{Float64}, Ptr{Float64}, Int64),
                    B.ctx.h, csr, a, x.p, o, res, λ, hist, length(hist)))
    end
    log ? (T(λ[]), x, history(res, hist, 0.0, 0.0)) : (T(λ[]), x)
end
invpowm!(B, x0; kwargs...) = powm!(B, x0; inverse = true, kwargs...)

# ------------------------------------------------------------------------------------------- stationary methods
# jacobi!(x, A, b; maxiter), gauss_seidel!, sor!(x, A, b, ω; maxiter), ssor!  src/stationary_sparse.jl:233-424
for (f, code, hasω) in ((:jacobi!, 0, false), (:gauss_seidel!, 1, false), (:sor!, 2, true), (:ssor!, 3, true))
    args = hasω ? (:(ω::Real),) : ()
    ωv = hasω ? :ω : 1.0
    @eval function IterativeSolvers.$f(x::B200Vector{T}, A::B200CSR{T}, b::B200Vector{T}, $(args...); maxiter::Int = 10) where {T}
        status = ccall((:b200_stationary, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Float64, Int64),
                       A.ctx.h, A.h, x.p, b.p, $code, $ωv, maxiter)
        status == -5 && throw(SingularException(0))            # DiagonalIndices  src/stationary_sparse.jl:19
        check(status); x
    end
end

Base.size(A::B200LinearOperator) = (A.m, A.n)
Base.size(A::B200LinearOperator, d::Integer) = d == 1 ? A.m : (d == 2 ? A.n : 1)

end # module
