# KrylovB200.jl -- the Julia face of the boundary: a storage type + operator type for which
# Krylov.jl's documented plugin points (docs/src/custom_workspaces.md:107,151-300) resolve to
# `ccall`s into libkrylov_b200.so.
#
# STATUS: Julia is not installed in the build image, so this file has never been executed here.
# It is the reference-side binding a maintainer would add (see INTEGRATION.md); everything it
# calls is exercised through the same C ABI by tests/ via ctypes, and tests/test_julia_binding.py
# parses every `ccall` below and checks symbol, argument count and argument/return types against
# include/krylov_b200.h, and the three mirrored structs (COpts, CExt, CStats) field by field.
#
# Two levels, as in the reference:
#   (1) primitive level  -- Krylov.kdot / knorm / kaxpy! / ... / kmul! overloads for B200Vector /
#       B200CSR.  Every solver of Krylov.jl then runs on the GPU unmodified (scalars come back to
#       the host by value, exactly like CuVector storage, src/krylov_utils.jl:309-349).
#   (2) solver level     -- cg!/gmres!/bicgstab!/minres! methods for workspaces whose storage is
#       B200Vector: one C call per solve, fused kernels, device-resident scalars.
module KrylovB200

using Krylov, LinearAlgebra, SparseArrays
import Krylov: kdot, kdotr, knorm, kscal!, kdiv!, kaxpy!, kaxpby!, kcopy!, kscalcopy!, kdivcopy!, kfill!, kmul!

const lib = get(ENV, "KRYLOV_B200_LIB", "libkrylov_b200.so")
const BlasT = Union{Float32, Float64}
dtype_id(::Type{Float32}) = Cint(0)
dtype_id(::Type{Float64}) = Cint(1)

# ---- execution context (one stream + reduction scratch), lazily created -------------------------
const CTX = Ref{Ptr{Cvoid}}(C_NULL)
function ctx()
  if CTX[] == C_NULL
    CTX[] = ccall((:kb200_ctx_create, lib), Ptr{Cvoid}, (Cint,), -1)
    CTX[] == C_NULL && error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
  end
  CTX[]
end
check(rc) = rc == 0 ? nothing : error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))

# ---- storage type: S <: AbstractVector{T} with length/similar/S(undef,n) (inplace.md:29-38) ------
mutable struct B200Vector{T<:BlasT} <: AbstractVector{T}
  ptr::Ptr{Cvoid}
  n::Int
  function B200Vector{T}(::UndefInitializer, n::Integer) where T
    p = n == 0 ? C_NULL : ccall((:kb200_alloc, lib), Ptr{Cvoid}, (Clonglong,), n * sizeof(T))
    v = new{T}(p, n)
    finalizer(x -> (x.ptr != C_NULL && ccall((:kb200_free, lib), Cint, (Ptr{Cvoid},), x.ptr); x.ptr = C_NULL), v)
    v
  end
end
function B200Vector(h::Vector{T}) where T<:BlasT
  v = B200Vector{T}(undef, length(h))
  check(ccall((:kb200_h2d, lib), Cint, (Ptr{Cvoid}, Ptr{T}, Clonglong), v.ptr, h, sizeof(h)))
  v
end
Base.size(v::B200Vector) = (v.n,)
Base.length(v::B200Vector) = v.n
Base.similar(v::B200Vector{T}) where T = B200Vector{T}(undef, v.n)
Base.similar(v::B200Vector, ::Type{T}, dims::Dims{1}) where T = B200Vector{T}(undef, dims[1])
Base.getindex(v::B200Vector, i::Int) = error("scalar indexing of a B200Vector is disabled (cf. CUDA.allowscalar(false))")
function Base.Vector(v::B200Vector{T}) where T
  h = Vector{T}(undef, v.n)
  check(ccall((:kb200_d2h, lib), Cint, (Ptr{T}, Ptr{Cvoid}, Clonglong), h, v.ptr, sizeof(h)))
  h
end

# ---- primitives: same signatures as src/krylov_utils.jl:309-347 ----------------------------------
function kdot(n::Integer, x::B200Vector{T}, y::B200Vector{T}) where T
  r = Ref{Cdouble}()
  check(ccall((:kb200_dot, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ref{Cdouble}), ctx(), dtype_id(T), n, x.ptr, y.ptr, r))
  T(r[])
end
kdotr(n::Integer, x::B200Vector{T}, y::B200Vector{T}) where T = kdot(n, x, y)
function knorm(n::Integer, x::B200Vector{T}) where T
  r = Ref{Cdouble}()
  check(ccall((:kb200_nrm2, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ref{Cdouble}), ctx(), dtype_id(T), n, x.ptr, r))
  T(r[])
end
kaxpy!(n::Integer, s::T, x::B200Vector{T}, y::B200Vector{T}) where T =
  (check(ccall((:kb200_axpy, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Cdouble, Ptr{Cvoid}, Ptr{Cvoid}), ctx(), dtype_id(T), n, s, x.ptr, y.ptr)); y)
kaxpby!(n::Integer, s::T, x::B200Vector{T}, t::T, y::B200Vector{T}) where T =
  (check(ccall((:kb200_axpby, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Cdouble, Ptr{Cvoid}, Cdouble, Ptr{Cvoid}), ctx(), dtype_id(T), n, s, x.ptr, t, y.ptr)); y)
kscal!(n::Integer, s::T, x::B200Vector{T}) where T =
  (check(ccall((:kb200_scal, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Cdouble, Ptr{Cvoid}), ctx(), dtype_id(T), n, s, x.ptr)); x)
kdiv!(n::Integer, x::B200Vector{T}, s::T) where T = kscal!(n, one(T) / s, x)          # krylov_utils.jl:325
kcopy!(n::Integer, y::B200Vector{T}, x::B200Vector{T}) where T =
  (check(ccall((:kb200_copy, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}), ctx(), dtype_id(T), n, y.ptr, x.ptr)); y)
kscalcopy!(n::Integer, y::B200Vector{T}, s::T, x::B200Vector{T}) where T =
  (check(ccall((:kb200_scalcopy, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Cdouble, Ptr{Cvoid}), ctx(), dtype_id(T), n, y.ptr, s, x.ptr)); y)
kdivcopy!(n::Integer, y::B200Vector{T}, x::B200Vector{T}, s::T) where T =
  (check(ccall((:kb200_divcopy, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Cdouble), ctx(), dtype_id(T), n, y.ptr, x.ptr, s)); y)
kfill!(x::B200Vector{T}, val::T) where T =
  (check(ccall((:kb200_fill, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Cdouble), ctx(), dtype_id(T), x.n, x.ptr, val)); x)

# ---- operator: CSR resident in HBM ------------------------------------------------------------------
mutable struct B200CSR{T<:BlasT}
  handle::Ptr{Cvoid}
  m::Int
  n::Int
  function B200CSR{T}(h::Ptr{Cvoid}, m::Integer, n::Integer) where T
    h == C_NULL && error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    op = new{T}(h, m, n)
    finalizer(o -> (o.handle != C_NULL && ccall((:kb200_csr_destroy, lib), Cvoid, (Ptr{Cvoid},), o.handle); o.handle = C_NULL), op)
    op
  end
end
# SparseMatrixCSC{T,Int64} is CSC, 1-based, Int64.  CSR(A) == CSC(A'): for the (symmetric) CG/MINRES
# operators the arrays can be passed as they are; for a general A pass the CSC arrays of copy(A').
function B200CSR(A::SparseMatrixCSC{T,Int64}; symmetric::Bool = size(A, 1) == size(A, 2) && issymmetric(A)) where T<:BlasT
  size(A, 1) == size(A, 2) || return rect_csr(A)
  At = symmetric ? A : SparseMatrixCSC(transpose(A))
  h = ccall((:kb200_csr_create, lib), Ptr{Cvoid},
            (Ptr{Cvoid}, Cint, Cint, Clonglong, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint, Cint),
            ctx(), dtype_id(T), size(A, 1), nnz(A), At.colptr, At.rowval, At.nzval, 1, 8, 0)
  B200CSR{T}(h, size(A)...)
end
# Rectangular A (LSQR / LSMR): the CSC arrays of A are the CSR arrays of A^T (n x m), so upload those as they are and
# let the library form A from them -- one transpose instead of one here and one in the library.
function rect_csr(A::SparseMatrixCSC{T,Int64}) where T<:BlasT
  m, n = size(A)
  ht = ccall((:kb200_csr_create_rect, lib), Ptr{Cvoid},
             (Ptr{Cvoid}, Cint, Cint, Cint, Clonglong, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint, Cint),
             ctx(), dtype_id(T), n, m, nnz(A), A.colptr, A.rowval, A.nzval, 1, 8, 0)
  At = B200CSR{T}(ht, n, m)
  adjoint(At)
end
# Matrix Market ingestion on the library side (benchmark/benchmarks.jl:23-33 reads SuiteSparse .mtx files)
function B200CSR(path::AbstractString, ::Type{T} = Float64) where T<:BlasT
  h = ccall((:kb200_csr_read_mtx, lib), Ptr{Cvoid}, (Ptr{Cvoid}, Cstring, Cint), ctx(), path, dtype_id(T))
  h == C_NULL && error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
  n = Ref{Cint}(0); nz = Ref{Clonglong}(0)
  check(ccall((:kb200_csr_info, lib), Cint, (Ptr{Cvoid}, Ref{Cint}, Ref{Clonglong}), h, n, nz))
  B200CSR{T}(h, n[], n[])
end
# A' : a new device-resident operator holding the transpose (= adjoint for the real types of this path), square or
# rectangular.  lsqr! / lsmr! on a B200CSR run natively (ls_solve! below; the library forms and caches A^T itself);
# the other methods of the family (BiLQ, QMR, CGLS, CRAIG, ...) reach A' through the primitive overloads, one `ccall`
# per k* operation (docs/src/matrix_free.md:36-44)
function Base.adjoint(A::B200CSR{T}) where T
  h = ccall((:kb200_csr_transpose, lib), Ptr{Cvoid}, (Ptr{Cvoid}, Ptr{Cvoid}), ctx(), A.handle)
  B200CSR{T}(h, A.n, A.m)
end
Base.transpose(A::B200CSR) = adjoint(A)
Base.size(A::B200CSR) = (A.m, A.n)
Base.size(A::B200CSR, i::Integer) = i == 1 ? A.m : (i == 2 ? A.n : 1)
Base.eltype(::B200CSR{T}) where T = T
kmul!(y::B200Vector{T}, A::B200CSR{T}, x::B200Vector{T}) where T =       # custom_workspaces.md:114-115
  (check(ccall((:kb200_spmv_csr, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint), ctx(), A.handle, x.ptr, y.ptr, 0)); y)
LinearAlgebra.mul!(y::B200Vector, A::B200CSR, x::B200Vector) = kmul!(y, A, x)

# ---- diagonal preconditioner resident in HBM (docs/src/preconditioners.md:33,159) ---------------------
# M = B200Diagonal(d): mul!(y, M, x) is y = d .* x;  with ldiv = true the solver applies x ./ d.
struct B200Diagonal{T<:BlasT}
  d::B200Vector{T}
end
Base.size(D::B200Diagonal) = (D.d.n, D.d.n)
Base.eltype(::B200Diagonal{T}) where T = T
# M = B200BlockDiagonal(bs, blocks): block-Jacobi, ceil(n / bs) dense bs x bs row-major blocks of the operator the
# solver applies (P^-1 with ldiv = false); cg! runs it inside the persistent fused kernel (include/krylov_b200.h)
struct B200BlockDiagonal{T<:BlasT}
  bs::Int
  blocks::B200Vector{T}
  n::Int
end
Base.size(D::B200BlockDiagonal) = (D.n, D.n)
Base.eltype(::B200BlockDiagonal{T}) where T = T

# ---- dense n x p block of right-hand sides / solutions resident in HBM (column-major, like Matrix) --------------
mutable struct B200Matrix{T<:BlasT} <: AbstractMatrix{T}
  ptr::Ptr{Cvoid}
  n::Int
  p::Int
  function B200Matrix{T}(::UndefInitializer, n::Integer, p::Integer) where T
    q = n * p == 0 ? C_NULL : ccall((:kb200_alloc, lib), Ptr{Cvoid}, (Clonglong,), n * p * sizeof(T))
    v = new{T}(q, n, p)
    finalizer(x -> (x.ptr != C_NULL && ccall((:kb200_free, lib), Cint, (Ptr{Cvoid},), x.ptr); x.ptr = C_NULL), v)
    v
  end
end
function B200Matrix(h::Matrix{T}) where T<:BlasT
  v = B200Matrix{T}(undef, size(h)...)
  check(ccall((:kb200_h2d, lib), Cint, (Ptr{Cvoid}, Ptr{T}, Clonglong), v.ptr, h, sizeof(h)))
  v
end
Base.size(v::B200Matrix) = (v.n, v.p)
Base.similar(v::B200Matrix{T}) where T = B200Matrix{T}(undef, v.n, v.p)
Base.getindex(v::B200Matrix, i::Int, j::Int) = error("scalar indexing of a B200Matrix is disabled")
function Base.Matrix(v::B200Matrix{T}) where T
  h = Matrix{T}(undef, v.n, v.p)
  check(ccall((:kb200_d2h, lib), Cint, (Ptr{T}, Ptr{Cvoid}, Clonglong), h, v.ptr, sizeof(h)))
  h
end

# ---- solver level: one C call per solve (fused kernels) ------------------------------------------------
# The workspace keeps Krylov.jl's type (CgWorkspace{T,T,B200Vector{T}}) for its stats and public fields; the
# device vectors of the fused solve live in a libkrylov_b200 workspace (KRYLOV_CUDA: device pointers) that is
# created ONCE per Krylov.jl workspace and kept in HANDLES, so an in-place solve allocates nothing
# (test/test_allocations.jl:54-57).
const SOLVER_ID = Dict(:cg => 0, :cr => 1, :minres => 3, :diom => 5, :dqgmres => 6, :fom => 7, :gmres => 8, :fgmres => 9,
                       :bicgstab => 10, :cgs => 11, :lslq => 20, :lsqr => 21, :lsmr => 22, :cgls => 24, :crls => 25, :bilq => 12, :qmr => 13,
                       :car => 32, :minares => 33, :trilqr => 18, :bilqr => 19, :craig => 28, :craigmr => 29, :lnlq => 30,
                       :cgne => 26, :crmr => 27, :cg_lanczos => 100)
struct COpts   # KrylovOptions, interfaces/src/c_enums.jl:40-62
  atol::Cdouble; rtol::Cdouble; itmax::Cint; verbose::Cint; lambda::Cdouble; tau::Cdouble; nu::Cdouble
  timemax::Cdouble; radius::Cdouble; restart::Cint; reorthogonalization::Cint; linesearch::Cint
end
struct CExt    # KrylovB200Options (include/krylov_b200.h)
  history::Cint; ldiv::Cint; etol::Cdouble; conlim::Cdouble; fused::Cint; batch::Cint
  callback::Ptr{Cvoid}; callback_user::Ptr{Cvoid}; time_kernels::Cint; check_curvature::Cint; cr_gamma::Cdouble
  axtol::Cdouble; btol::Cdouble; sigma::Cdouble; utol::Cdouble; transfer_to_lsqr::Cint; transfer_to_bicg::Cint
end
struct CStats  # KrylovB200Stats (include/krylov_b200.h)
  niter::Cint; solved::Cint; inconsistent::Cint; indefinite::Cint; npcCount::Cint
  nresiduals::Cint; nAresiduals::Cint; nAcond::Cint
  allocation_timer::Cdouble; timer::Cdouble; status::NTuple{96,UInt8}; Anorm::Cdouble
  error_with_bnd::Cint; nerr_lbnds::Cint; nerr_ubnds_lq::Cint; nerr_ubnds_cg::Cint
  solved_primal::Cint; solved_dual::Cint; nresiduals_dual::Cint
end

mutable struct Handle
  ptr::Ptr{Cvoid}
  op::Ptr{Cvoid}          # CSR object currently attached
  block::Bool             # krylov_block_* handle (block_gmres!)
end
const HANDLES = IdDict{Any,Handle}()
function handle_for(method::Symbol, ws, A::B200CSR{T}, memory::Int, window::Int) where T
  h = get(HANDLES, ws, nothing)
  if h === nothing
    out = Ref{Ptr{Cvoid}}(C_NULL)
    wo = Ref((Cint(memory), Cint(window)))            # KrylovWorkspaceOptions {memory, window}
    rc = ccall((:krylov_workspace_create, lib), Cint, (Cint, Cint, Cint, Cint, Cint, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}),
               SOLVER_ID[method], A.m, A.n, dtype_id(T), 1, wo, out)
    rc == 0 || error("krylov_workspace_create -> $rc: " * unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    h = Handle(out[], C_NULL, false)
    finalizer(x -> (x.ptr != C_NULL && ccall((:krylov_workspace_free, lib), Cint, (Ptr{Cvoid},), x.ptr); x.ptr = C_NULL), h)
    HANDLES[ws] = h
  end
  if h.op != A.handle      # operator resident in HBM: attach, no copy
    check(ccall((:krylov_b200_attach_csr, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, A.handle))
    h.op = A.handle
  end
  h
end

# callback trampoline: int (*)(void *ws, void *user); `user` carries the Julia closure and the Krylov.jl workspace
function _cb_tramp(_c_ws::Ptr{Cvoid}, user::Ptr{Cvoid})::Cint
  f, ws = unsafe_pointer_to_objref(user)::Tuple{Any,Any}
  r = f(ws)
  r isa Bool || throw(TypeError(:callback, "", Bool, r))   # cg.jl:264, test_cg.jl:130
  Cint(r)
end

function set_precond!(h::Handle, which::Int, ::UniformScaling)
  check(ccall((:krylov_b200_set_preconditioner_diag, lib), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Cint), h.ptr, which, C_NULL, 0))
  h.block || check(ccall((:krylov_b200_set_preconditioner_blockdiag, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Cint), h.ptr, which, 0, C_NULL, 0))
  nothing
end
set_precond!(h::Handle, which::Int, D::B200Diagonal) =
  check(ccall((:krylov_b200_set_preconditioner_diag, lib), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Cint), h.ptr, which, D.d.ptr, 1))
function set_precond!(h::Handle, which::Int, D::B200BlockDiagonal)
  check(ccall((:krylov_b200_set_preconditioner_diag, lib), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Cint), h.ptr, which, C_NULL, 0))
  check(ccall((:krylov_b200_set_preconditioner_blockdiag, lib), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Cint), h.ptr, which, D.bs, D.blocks.ptr, 1))
end
set_precond!(::Handle, ::Int, P) = error("libkrylov_b200: preconditioners must be I or a B200Diagonal (got $(typeof(P))); " *
                                         "any other operator runs through the primitive overloads (generic Krylov.jl method)")

function fill_stats!(ws, h::Handle, ::Type{T}) where T
  cs = Ref{CStats}()
  check(ccall((:krylov_b200_get_stats, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, cs))
  s = cs[]
  st = ws.stats
  st.niter = s.niter; st.solved = s.solved != 0; st.inconsistent = s.inconsistent != 0
  st.timer = s.timer
  hasproperty(st, :allocation_timer) && (st.allocation_timer = s.allocation_timer)
  hasproperty(st, :indefinite) && (st.indefinite = s.indefinite != 0)
  hasproperty(st, :npcCount) && (st.npcCount = s.npcCount)
  hasproperty(st, :Anorm) && (st.Anorm = T(s.Anorm))            # LanczosStats (cg_lanczos!)
  hasproperty(st, :error_with_bnd) && (st.error_with_bnd = s.error_with_bnd != 0)   # LSLQStats, LNLQStats
  bytes = collect(s.status); z = findfirst(==(0x00), bytes)
  st.status = String(bytes[1:(z === nothing ? length(bytes) : z - 1)])
  for (which, field, cnt) in ((0, :residuals, s.nresiduals), (1, :Aresiduals, s.nAresiduals), (2, :Acond, s.nAcond),
                              (3, :err_lbnds, s.nerr_lbnds), (4, :err_ubnds_lq, s.nerr_ubnds_lq), (5, :err_ubnds_cg, s.nerr_ubnds_cg),
                              (3, :error_bnd_x, s.nerr_lbnds), (4, :error_bnd_y, s.nerr_ubnds_lq))   # LNLQStats
    hasproperty(st, field) || continue
    buf = Vector{Cdouble}(undef, cnt)
    got = cnt == 0 ? 0 : ccall((:krylov_b200_get_history, lib), Cint, (Ptr{Cvoid}, Cint, Ptr{Cdouble}, Cint), h.ptr, which, buf, cnt)
    v = getproperty(st, field); empty!(v); append!(v, T.(buf[1:got]))
  end
  st
end

# kwargs: the union of cg.jl:100-111, minres.jl:138-151, gmres.jl:96-108, bicgstab.jl:105-116, car.jl:90-99 and
# minares.jl:93-104 (a solver ignores the ones it does not have, exactly like the C layer's option families,
# interfaces/src/c_stores.jl:287-398); MINARES's Artol travels in the axtol field of the extended options
function fused_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}; c::Union{Nothing,B200Vector{T}} = nothing,
                      M = I, N = I, ldiv::Bool = false, atol::T = √eps(T), rtol::T = √eps(T), etol::T = √eps(T),
                      conlim::T = 1 / √eps(T), itmax::Int = 0, timemax::Float64 = Inf, verbose::Int = 0,
                      history::Bool = false, callback = workspace -> false, iostream::IO = stdout,
                      radius::T = zero(T), linesearch::Bool = false, λ::T = zero(T), γ::T = √eps(T),
                      check_curvature::Bool = false, restart::Bool = false, reorthogonalization::Bool = false,
                      memory::Int = 0, window::Int = 0, Artol::T = √eps(T)) where T
  A.m == A.n || error("System must be square")
  length(b) == A.m || error("Inconsistent problem size")
  h = handle_for(method, ws, A, memory, window)
  set_precond!(h, 0, M)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, etol, conlim, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, check_curvature, γ, Artol, NaN, 0.0, NaN, 0, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, λ, NaN, NaN, isinf(timemax) ? NaN : timemax, radius, restart, reorthogonalization, linesearch))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    if ws.warm_start                      # warm_start!(ws, x0) stored x0 in ws.Δx (workspace_accessors.jl:193-200)
      check(ccall((:krylov_warm_start, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.Δx.ptr, A.n))
      ws.warm_start = false
    end
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, c === nothing ? C_NULL : c.ptr, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    # solution(ws) is ws.x itself (workspace_accessors.jl:149): device-to-device copy into the Krylov.jl vector
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
  end
  fill_stats!(ws, h, T)
  ws
end

# x0 as optional positional argument = warm_start! + solve (cg.jl:98, def_optargs_cg)
function fused_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}, x0::B200Vector{T}; kw...) where T
  Krylov.warm_start!(ws, x0)
  fused_solve!(method, ws, A, b; kw...)
end

for (fn, WS, sym, memexpr) in ((:cg!, :CgWorkspace, :cg, :(0)),
                               (:gmres!, :GmresWorkspace, :gmres, :(length(ws.c))), (:bicgstab!, :BicgstabWorkspace, :bicgstab, :(0)),
                               # sibling solvers served by the same library (SURVEY.md 8f-3); every other method keeps
                               # running through the k* overloads above, one kernel per call
                               (:cr!, :CrWorkspace, :cr, :(0)), (:cgs!, :CgsWorkspace, :cgs, :(0)),
                               (:cg_lanczos!, :CgLanczosWorkspace, :cg_lanczos, :(0)), (:fom!, :FomWorkspace, :fom, :(length(ws.l))),
                               (:fgmres!, :FgmresWorkspace, :fgmres, :(length(ws.c))), (:dqgmres!, :DqgmresWorkspace, :dqgmres, :(length(ws.V))),
                               (:diom!, :DiomWorkspace, :diom, :(length(ws.V))),
                               # car! (M only) and minares! (λ, Artol; no preconditioner): fused passes on a B200CSR
                               (:car!, :CarWorkspace, :car, :(0)), (:minares!, :MinaresWorkspace, :minares, :(0)))
  @eval begin
    Krylov.$fn(ws::Krylov.$WS{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
      fused_solve!($(QuoteNode(sym)), ws, A, b; memory = $memexpr, kw...)
    Krylov.$fn(ws::Krylov.$WS{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}, x0::B200Vector{T}; kw...) where T =
      fused_solve!($(QuoteNode(sym)), ws, A, b, x0; memory = $memexpr, kw...)
  end
end
# MINRES keeps `window` in the length of its err_vec (krylov_workspaces.jl:121-127)
Krylov.minres!(ws::Krylov.MinresWorkspace{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  fused_solve!(:minres, ws, A, b; window = length(ws.err_vec), kw...)
Krylov.minres!(ws::Krylov.MinresWorkspace{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}, x0::B200Vector{T}; kw...) where T =
  fused_solve!(:minres, ws, A, b, x0; window = length(ws.err_vec), kw...)

# ---- lsqr! / lsmr! (src/lsqr.jl:142-162, src/lsmr.jl:146-166) on a rectangular B200CSR: one krylov_solve per solve ----
# The fused Golub-Kahan passes run when M = N = I and radius = 0; B200Diagonal M (m entries) / N (n entries) and the
# trust region run the library's primitive path.
function ls_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}; M = I, N = I, ldiv::Bool = false, sqd::Bool = false,
                   λ::T = zero(T), radius::T = zero(T), etol::T = √eps(T), axtol::T = √eps(T), btol::T = √eps(T),
                   conlim::T = 1 / √eps(T), atol::T = zero(T), rtol::T = zero(T), itmax::Int = 0, timemax::Float64 = Inf,
                   verbose::Int = 0, history::Bool = false, callback = workspace -> false, iostream::IO = stdout) where T
  length(b) == A.m || error("Inconsistent problem size")
  sqd && (λ ≠ 0) && error("sqd cannot be set to true if λ ≠ 0 !")
  sqd && (λ = one(T))
  h = handle_for(method, ws, A, 0, length(ws.err_vec))
  set_precond!(h, 0, M)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, etol, conlim, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, axtol, btol, 0.0, NaN, 0, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, λ, NaN, NaN, isinf(timemax) ? NaN : timemax, radius, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, C_NULL, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
  end
  fill_stats!(ws, h, T)
  ws
end
Krylov.lsqr!(ws::Krylov.LsqrWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  ls_solve!(:lsqr, ws, A, b; kw...)
Krylov.lsmr!(ws::Krylov.LsmrWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  ls_solve!(:lsmr, ws, A, b; kw...)

# ---- lslq! (src/lslq.jl:178-196) on a rectangular B200CSR: one krylov_solve per solve ----
# Its own kwargs and defaults (atol = rtol = √eps(T), σ, utol, transfer_to_lsqr, no radius); B200Diagonal M (m entries)
# and N (n entries).  The fused Golub-Kahan passes run when M = N = I.
function lslq_solve!(ws, A::B200CSR{T}, b::B200Vector{T}; M = I, N = I, ldiv::Bool = false, transfer_to_lsqr::Bool = false,
                     sqd::Bool = false, λ::T = zero(T), σ::T = zero(T), etol::T = √eps(T), utol::T = √eps(T),
                     btol::T = √eps(T), conlim::T = 1/√eps(T), atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0,
                     timemax::Float64 = Inf, verbose::Int = 0, history::Bool = false, callback = workspace -> false,
                     iostream::IO = stdout) where T
  length(b) == A.m || error("Inconsistent problem size")
  sqd && (λ ≠ 0) && error("sqd cannot be set to true if λ ≠ 0 !")
  sqd && (λ = one(T))
  h = handle_for(:lslq, ws, A, 0, length(ws.err_vec))
  set_precond!(h, 0, M)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, etol, conlim, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, btol, σ, utol,
                 transfer_to_lsqr, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, λ, NaN, NaN, isinf(timemax) ? NaN : timemax, 0, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, C_NULL, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
  end
  fill_stats!(ws, h, T)
  ws
end
Krylov.lslq!(ws::Krylov.LslqWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  lslq_solve!(ws, A, b; kw...)

# ---- cgls! / crls! (src/cgls.jl:110-121, src/crls.jl:101-112) on a rectangular B200CSR: one krylov_solve per solve ----
# Their own kwargs and defaults (atol = rtol = √eps(T)); M acts on the m-dimensional residual space (a B200Diagonal of
# m entries) and there is no N.  The fused passes run when M = I and radius = 0.
function normal_ls_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}; M = I, ldiv::Bool = false,
                          radius::T = zero(T), λ::T = zero(T), atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0,
                          timemax::Float64 = Inf, verbose::Int = 0, history::Bool = false, callback = workspace -> false,
                          iostream::IO = stdout) where T
  length(b) == A.m || error("Inconsistent problem size")
  h = handle_for(method, ws, A, 0, 0)
  set_precond!(h, 0, M)
  set_precond!(h, 1, I)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, NaN, NaN, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, NaN, 0.0, NaN, 0, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, λ, NaN, NaN, isinf(timemax) ? NaN : timemax, radius, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, C_NULL, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
  end
  fill_stats!(ws, h, T)
  ws
end
Krylov.cgls!(ws::Krylov.CglsWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  normal_ls_solve!(:cgls, ws, A, b; kw...)
Krylov.crls!(ws::Krylov.CrlsWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  normal_ls_solve!(:crls, ws, A, b; kw...)

# ---- craig! / craigmr! (src/craig.jl:151-166, src/craigmr.jl:141-153) on a rectangular B200CSR: one krylov_solve ----
# The least-norm solution of A x = b with x = Aᵀ y: the workspace's x receives x and its y the multipliers y.  The
# library forms Aᵀ once per operator; the fused Golub-Kahan passes run when M = N = I and λ = 0, B200Diagonal M
# (m entries) / N (n entries) and λ > 0 run its primitive path.  btol, conlim and transfer_to_lsqr are CRAIG's only.
function leastnorm_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}; M = I, N = I, ldiv::Bool = false,
                          transfer_to_lsqr::Bool = false, sqd::Bool = false, λ::T = zero(T), btol::T = √eps(T),
                          conlim::T = 1/√eps(T), atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0,
                          timemax::Float64 = Inf, verbose::Int = 0, history::Bool = false, callback = workspace -> false,
                          iostream::IO = stdout) where T
  length(b) == A.m || error("Inconsistent problem size")
  sqd && (λ ≠ 0) && error("sqd cannot be set to true if λ ≠ 0 !")
  sqd && (λ = one(T))
  h = handle_for(method, ws, A, 0, 0)
  set_precond!(h, 0, M)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, NaN, conlim, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, btol, 0.0, NaN,
                 transfer_to_lsqr, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, λ, NaN, NaN, isinf(timemax) ? NaN : timemax, 0.0, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, C_NULL, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
    check(ccall((:krylov_get_y, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.y.ptr, A.m))
  end
  fill_stats!(ws, h, T)
  ws
end
Krylov.craig!(ws::Krylov.CraigWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  leastnorm_solve!(:craig, ws, A, b; kw...)
Krylov.craigmr!(ws::Krylov.CraigmrWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  leastnorm_solve!(:craigmr, ws, A, b; kw...)

# ---- lnlq! (src/lnlq.jl:144-160) on a rectangular B200CSR: one krylov_solve ----
# A sibling of leastnorm_solve!, whose kwargs are CRAIG's and CRAIGMR's.  The fused Golub-Kahan passes run when
# M = N = I and λ = 0.  The extended options carry σ in `sigma`, utolx in `utol`, utoly in `etol` and transfer_to_craig
# in `transfer_to_bicg`; the bounds come back in stats.error_bnd_x / error_bnd_y (history slots 3 and 4).
function lnlq_solve!(ws, A::B200CSR{T}, b::B200Vector{T}; M = I, N = I, ldiv::Bool = false, transfer_to_craig::Bool = true,
                     sqd::Bool = false, λ::T = zero(T), σ::T = zero(T), utolx::T = √eps(T), utoly::T = √eps(T),
                     atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0, timemax::Float64 = Inf, verbose::Int = 0,
                     history::Bool = false, callback = workspace -> false, iostream::IO = stdout) where T
  length(b) == A.m || error("Inconsistent problem size")
  sqd && (λ ≠ 0) && error("sqd cannot be set to true if λ ≠ 0 !")
  sqd && (λ = one(T))
  h = handle_for(:lnlq, ws, A, 0, 0)
  set_precond!(h, 0, M)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, utoly, NaN, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, NaN, σ, utolx,
                 0, transfer_to_craig))
  o = Ref(COpts(atol, rtol, itmax, verbose, λ, NaN, NaN, isinf(timemax) ? NaN : timemax, 0.0, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, C_NULL, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
    check(ccall((:krylov_get_y, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.y.ptr, A.m))
  end
  fill_stats!(ws, h, T)
  ws
end
Krylov.lnlq!(ws::Krylov.LnlqWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  lnlq_solve!(ws, A, b; kw...)

# ---- cgne! / crmr! (src/cgne.jl:113-131, src/crmr.jl:111-129) on a rectangular B200CSR: one krylov_solve ----------
# A sibling of normal_ls_solve! and leastnorm_solve!, whose kwargs are CGLS's / CRLS's and CRAIG's / CRAIGMR's.  CG and
# CR on A Aᵀ y = b with x = Aᵀ y; only x comes back.  N acts on the m-dimensional residual space (a B200Diagonal of m
# entries) and there is no M.  The fused passes run when N = I and λ = 0.
function normal_ln_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}; N = I, ldiv::Bool = false, λ::T = zero(T),
                          atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0, timemax::Float64 = Inf, verbose::Int = 0,
                          history::Bool = false, callback = workspace -> false, iostream::IO = stdout) where T
  length(b) == A.m || error("Inconsistent problem size")
  h = handle_for(method, ws, A, 0, 0)
  set_precond!(h, 0, I)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, NaN, NaN, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, NaN, 0.0, NaN, 0, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, λ, NaN, NaN, isinf(timemax) ? NaN : timemax, 0.0, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, C_NULL, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
  end
  fill_stats!(ws, h, T)
  ws
end
Krylov.cgne!(ws::Krylov.CgneWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  normal_ln_solve!(:cgne, ws, A, b; kw...)
Krylov.crmr!(ws::Krylov.CrmrWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  normal_ln_solve!(:crmr, ws, A, b; kw...)

# ---- bilq! / qmr! (src/bilq.jl:97-115, src/qmr.jl:104-114) on a square B200CSR: one krylov_solve per solve ------------
# The library forms Aᵀ once per operator and runs the fused Lanczos biorthogonalization when M = N = I; `c` defaults to b.
function biorth_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}; c::B200Vector{T} = b,
                       transfer_to_bicg::Bool = true, M = I, N = I, ldiv::Bool = false, atol::T = √eps(T),
                       rtol::T = √eps(T), itmax::Int = 0, timemax::Float64 = Inf, verbose::Int = 0, history::Bool = false,
                       callback = workspace -> false, iostream::IO = stdout) where T
  A.m == A.n || error("System must be square")
  length(b) == A.m || error("Inconsistent problem size")
  h = handle_for(method, ws, A, 0, 0)
  set_precond!(h, 0, M)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, NaN, NaN, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, NaN, 0.0, NaN, 0,
                 transfer_to_bicg))
  o = Ref(COpts(atol, rtol, itmax, verbose, 0.0, NaN, NaN, isinf(timemax) ? NaN : timemax, 0.0, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    if ws.warm_start                      # warm_start!(ws, x0) stored x0 in ws.Δx
      check(ccall((:krylov_warm_start, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.Δx.ptr, A.n))
      ws.warm_start = false
    end
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, c.ptr, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
  end
  fill_stats!(ws, h, T)
  ws
end
Krylov.bilq!(ws::Krylov.BilqWorkspace{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  biorth_solve!(:bilq, ws, A, b; kw...)
Krylov.qmr!(ws::Krylov.QmrWorkspace{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}; kw...) where T =
  biorth_solve!(:qmr, ws, A, b; kw...)

# ---- bilqr! / trilqr! (src/bilqr.jl:99-113, src/trilqr.jl:98-112) on a B200CSR: one krylov_solve per solve ----------
# A x = b and Aᵀ y = c together; the library forms Aᵀ once per operator and runs the fused passes.  TriLQR's
# transfer_to_usymcg travels in the transfer_to_bicg field of the extended options.  The workspace's y receives y, its
# stats (AdjointStats, src/krylov_stats.jl:263-280) both flags and both histories.
function adjoint_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}, c::B200Vector{T};
                        transfer_to_bicg::Bool = true, transfer_to_usymcg::Bool = true, atol::T = √eps(T),
                        rtol::T = √eps(T), itmax::Int = 0, timemax::Float64 = Inf, verbose::Int = 0, history::Bool = false,
                        callback = workspace -> false, iostream::IO = stdout) where T
  method === :bilqr && A.m != A.n && error("Systems must be square")
  length(b) == A.m || error("Inconsistent problem size")
  length(c) == A.n || error("Inconsistent problem size")
  h = handle_for(method, ws, A, 0, 0)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  transfer = method === :bilqr ? transfer_to_bicg : transfer_to_usymcg
  ext = Ref(CExt(history, false, NaN, NaN, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, NaN, 0.0, NaN, 0,
                 transfer))
  o = Ref(COpts(atol, rtol, itmax, verbose, 0.0, NaN, NaN, isinf(timemax) ? NaN : timemax, 0.0, 0, 0, 0))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    if ws.warm_start                      # warm_start!(ws, x0, y0) stored them in ws.Δx and ws.Δy
      check(ccall((:krylov_warm_start2, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint), h.ptr, ws.Δx.ptr,
                  ws.Δy.ptr, A.n, A.m))
      ws.warm_start = false
    end
    rc = ccall((:krylov_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, C_NULL, b.ptr, c.ptr, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_get_x, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.x.ptr, A.n))
    check(ccall((:krylov_get_y, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), h.ptr, ws.y.ptr, A.m))
  end
  fill_adjoint_stats!(ws, h, T)
  ws
end
function fill_adjoint_stats!(ws, h::Handle, ::Type{T}) where T
  cs = Ref{CStats}()
  check(ccall((:krylov_b200_get_stats, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, cs))
  s = cs[]
  st = ws.stats
  st.niter = s.niter; st.solved_primal = s.solved_primal != 0; st.solved_dual = s.solved_dual != 0; st.timer = s.timer
  bytes = collect(s.status); z = findfirst(==(0x00), bytes)
  st.status = String(bytes[1:(z === nothing ? length(bytes) : z - 1)])
  for (which, field, cnt) in ((0, :residuals_primal, s.nresiduals), (6, :residuals_dual, s.nresiduals_dual))
    buf = Vector{Cdouble}(undef, cnt)
    got = cnt == 0 ? 0 : ccall((:krylov_b200_get_history, lib), Cint, (Ptr{Cvoid}, Cint, Ptr{Cdouble}, Cint), h.ptr, which, buf, cnt)
    v = getproperty(st, field); empty!(v); append!(v, T.(buf[1:got]))
  end
  st
end
Krylov.bilqr!(ws::Krylov.BilqrWorkspace{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}, c::B200Vector{T}; kw...) where T =
  adjoint_solve!(:bilqr, ws, A, b, c; kw...)
Krylov.trilqr!(ws::Krylov.TrilqrWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T}, c::B200Vector{T};
               kw...) where T =
  adjoint_solve!(:trilqr, ws, A, b, c; kw...)

# ---- block_gmres! (src/block_gmres.jl:78-110; C ABI krylov.h:250-285): one krylov_block_solve per solve ------------------
# B, X, X0 are column-major n x p device matrices; the library keeps row-major panels internally and runs the
# tall-skinny products of Float64 p = 8 / 16 / 32 on the FP64 tensor cores.
function block_handle_for(ws, A::B200CSR{T}, p::Int, memory::Int) where T
  h = get(HANDLES, ws, nothing)
  if h === nothing
    out = Ref{Ptr{Cvoid}}(C_NULL)
    wo = Ref((Cint(memory), Cint(0)))
    rc = ccall((:krylov_block_workspace_create, lib), Cint, (Cint, Cint, Cint, Cint, Cint, Cint, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}),
               0, A.m, A.n, p, dtype_id(T), 1, wo, out)             # KRYLOV_BLOCK_GMRES = 0, KRYLOV_CUDA = 1
    rc == 0 || error("krylov_block_workspace_create -> $rc: " * unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    h = Handle(out[], C_NULL, true)
    finalizer(x -> (x.ptr != C_NULL && ccall((:krylov_block_workspace_free, lib), Cint, (Ptr{Cvoid},), x.ptr); x.ptr = C_NULL), h)
    HANDLES[ws] = h
  end
  if h.op != A.handle
    check(ccall((:krylov_b200_attach_csr, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, A.handle))
    h.op = A.handle
  end
  h
end

function Krylov.block_gmres!(ws::Krylov.BlockGmresWorkspace{T,T,B200Vector{T},B200Matrix{T}}, A::B200CSR{T}, B::B200Matrix{T};
                             M = I, N = I, ldiv::Bool = false, restart::Bool = false, reorthogonalization::Bool = false,
                             atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0, timemax::Float64 = Inf, verbose::Int = 0,
                             history::Bool = false, callback = workspace -> false, iostream::IO = stdout) where T
  A.m == A.n || error("System must be square")
  size(B, 1) == A.n || error("Inconsistent problem size")
  p = size(B, 2)
  h = block_handle_for(ws, A, p, length(ws.V))
  set_precond!(h, 0, M)
  set_precond!(h, 1, N)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, NaN, NaN, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, 0, NaN, NaN, NaN, 0.0, NaN, 0, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, 0.0, NaN, NaN, isinf(timemax) ? NaN : timemax, 0.0, restart, reorthogonalization, false))
  GC.@preserve user ext o begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    if ws.warm_start                      # warm_start!(ws, X0) stored X0 in ws.ΔX
      check(ccall((:krylov_block_warm_start, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint), h.ptr, ws.ΔX.ptr, A.n, p))
      ws.warm_start = false
    end
    rc = ccall((:krylov_block_solve, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, B.ptr, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    check(ccall((:krylov_block_get_X, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint), h.ptr, ws.X.ptr, A.n, p))
  end
  fill_stats!(ws, h, T)
  ws
end
function Krylov.block_gmres!(ws::Krylov.BlockGmresWorkspace{T,T,B200Vector{T},B200Matrix{T}}, A::B200CSR{T}, B::B200Matrix{T},
                             X0::B200Matrix{T}; kw...) where T
  Krylov.warm_start!(ws, X0)
  Krylov.block_gmres!(ws, A, B; kw...)
end

# ---- cg_lanczos_shift! / cgls_lanczos_shift! (src/cg_lanczos_shift.jl, src/cgls_lanczos_shift.jl): one shift handle per
# workspace (include/krylov_b200.h, krylov_b200_shift_*), one krylov_b200_shift_solve per solve; ws.x[i] is filled by a
# device-to-device copy and the LanczosShiftStats by one stats call and one history call per shift.
const SHIFT_ID = Dict(:cg_lanczos_shift => 101, :cgls_lanczos_shift => 102)
function shift_handle_for(method::Symbol, ws, A::B200CSR{T}, nshifts::Int) where T
  h = get(HANDLES, ws, nothing)
  if h === nothing
    out = Ref{Ptr{Cvoid}}(C_NULL)
    rc = ccall((:krylov_b200_shift_workspace_create, lib), Cint, (Cint, Cint, Cint, Cint, Cint, Cint, Ptr{Ptr{Cvoid}}),
               SHIFT_ID[method], A.m, A.n, nshifts, dtype_id(T), 1, out)                # KRYLOV_CUDA = 1
    rc == 0 || error("krylov_b200_shift_workspace_create -> $rc: " * unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    h = Handle(out[], C_NULL, false)
    finalizer(x -> (x.ptr != C_NULL && ccall((:krylov_b200_shift_workspace_free, lib), Cint, (Ptr{Cvoid},), x.ptr); x.ptr = C_NULL), h)
    HANDLES[ws] = h
  end
  if h.op != A.handle
    check(ccall((:krylov_b200_attach_csr, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, A.handle))
    h.op = A.handle
  end
  h
end

function shift_solve!(method::Symbol, ws, A::B200CSR{T}, b::B200Vector{T}, shifts::AbstractVector{T}, M, ldiv::Bool,
                      check_curvature::Bool, atol::T, rtol::T, itmax::Int, timemax::Float64, verbose::Int, history::Bool,
                      callback) where T
  nshifts = length(shifts)
  nshifts == ws.nshifts || error("workspace.nshifts = $(ws.nshifts) is inconsistent with length(shifts) = $nshifts")
  h = shift_handle_for(method, ws, A, nshifts)
  set_precond!(h, 0, M)
  user = Ref{Any}((callback, ws))
  cb = @cfunction(_cb_tramp, Cint, (Ptr{Cvoid}, Ptr{Cvoid}))
  ext = Ref(CExt(history, ldiv, NaN, NaN, 1, 0, cb, Base.unsafe_convert(Ptr{Cvoid}, user), 0, check_curvature, NaN, NaN, NaN, 0.0, NaN, 0, 1))
  o = Ref(COpts(atol, rtol, itmax, verbose, 0.0, NaN, NaN, isinf(timemax) ? NaN : timemax, 0.0, false, false, false))
  sh = Cdouble.(shifts)
  GC.@preserve user ext o sh begin
    check(ccall((:krylov_b200_set_options, lib), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, ext))
    rc = ccall((:krylov_b200_shift_solve, lib), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cdouble}, Ptr{Cvoid}, Ptr{Cvoid}),
               h.ptr, C_NULL, C_NULL, C_NULL, b.ptr, sh, C_NULL, o)
    rc == 0 || error(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())))
    for i in 1:nshifts
      check(ccall((:krylov_b200_shift_get_x, lib), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Cint), h.ptr, i - 1, ws.x[i].ptr, A.n))
    end
  end
  niter, solved, timer = Ref{Cint}(0), Ref{Cint}(0), Ref{Cdouble}(0)
  status = Vector{UInt8}(undef, 96)
  indef, hlen = Vector{Cint}(undef, nshifts), Vector{Cint}(undef, nshifts)
  check(ccall((:krylov_b200_shift_get_stats, lib), Cint,
              (Ptr{Cvoid}, Ptr{Cint}, Ptr{Cint}, Ptr{Cdouble}, Ptr{UInt8}, Cint, Ptr{Cint}, Ptr{Cint}),
              h.ptr, niter, solved, timer, status, 96, indef, hlen))
  st = ws.stats                                   # LanczosShiftStats (src/krylov_stats.jl:169-179)
  st.niter = niter[]; st.solved = solved[] != 0; st.timer = timer[]
  z = findfirst(==(0x00), status)
  st.status = String(status[1:(z === nothing ? length(status) : z - 1)])
  for i in 1:nshifts
    st.indefinite[i] = indef[i] != 0
    buf = Vector{Cdouble}(undef, hlen[i])
    got = hlen[i] == 0 ? 0 : ccall((:krylov_b200_shift_get_history, lib), Cint, (Ptr{Cvoid}, Cint, Ptr{Cdouble}, Cint),
                                   h.ptr, i - 1, buf, hlen[i])
    empty!(st.residuals[i]); append!(st.residuals[i], T.(buf[1:got]))
  end
  ws
end

# keywords: def_kwargs_cg_lanczos_shift (src/cg_lanczos_shift.jl:89-99)
function Krylov.cg_lanczos_shift!(ws::Krylov.CgLanczosShiftWorkspace{T,T,B200Vector{T}}, A::B200CSR{T}, b::B200Vector{T},
                                  shifts::AbstractVector{T}; M = I, ldiv::Bool = false, check_curvature::Bool = false,
                                  atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0, timemax::Float64 = Inf,
                                  verbose::Int = 0, history::Bool = false, callback = workspace -> false,
                                  iostream::IO = stdout) where T
  A.m == A.n || error("System must be square")
  length(b) == A.n || error("Inconsistent problem size")
  shift_solve!(:cg_lanczos_shift, ws, A, b, shifts, M, ldiv, check_curvature, atol, rtol, itmax, timemax, verbose, history, callback)
end

# keywords: def_kwargs_cgls_lanczos_shift (src/cgls_lanczos_shift.jl:91-100); M other than I is refused by the library
function Krylov.cgls_lanczos_shift!(ws::Krylov.CglsLanczosShiftWorkspace{T,T,B200Vector{T},B200Vector{T}}, A::B200CSR{T},
                                    b::B200Vector{T}, shifts::AbstractVector{T}; M = I, ldiv::Bool = false,
                                    atol::T = √eps(T), rtol::T = √eps(T), itmax::Int = 0, timemax::Float64 = Inf,
                                    verbose::Int = 0, history::Bool = false, callback = workspace -> false,
                                    iostream::IO = stdout) where T
  M === I || error("Preconditioner `M` is not supported.")
  length(b) == A.m || error("Inconsistent problem size")
  shift_solve!(:cgls_lanczos_shift, ws, A, b, shifts, M, ldiv, false, atol, rtol, itmax, timemax, verbose, history, callback)
end

# ---- Krylov processes (src/krylov_processes.jl): one kb200_<process> call each, every step enqueued on the GPU with the
# coefficients kept on the device and read back once (DESIGN.md §3i).  Bases come back as B200Matrix{T} (column-major,
# k + 1 columns), T / Tᴴ / L as SparseMatrixCSC{T,Int} with the reference's colptr / rowval, H as a dense Matrix{T}.
# Aᵀ (golub_kahan, nonhermitian_lanczos, saunders_simon_yip) is formed by the library for the call, through the host:
# those three copy the operator down once more before their single coefficient read-back.
proc_flags(allow_breakdown::Bool, reorthogonalization::Bool = false) = Cint(allow_breakdown) | (reorthogonalization ? Cint(2) : Cint(0))
# error(...) with the reference's message (the library prefixes its entry point's name)
proc_check(rc, name::String) = rc == 0 ? nothing :
  error(replace(unsafe_string(ccall((:krylov_b200_last_error, lib), Cstring, ())), "kb200_$name: " => ""; count = 1))

function tridiagonal_pattern(k::Int)            # krylov_processes.jl:35-51: (k+1) x k, 3k-1 stored entries
  colptr = zeros(Int, k+1); rowval = zeros(Int, 3k-1)
  colptr[1] = 1
  for i = 1:k
    pos = colptr[i]
    colptr[i+1] = 3i
    if i == 1
      rowval[pos] = i; rowval[pos+1] = i+1
    else
      rowval[pos] = i-1; rowval[pos+1] = i; rowval[pos+2] = i+1
    end
  end
  colptr, rowval
end

function bidiagonal_pattern(k::Int)             # krylov_processes.jl:331-346: (k+1) x (k+1), 2k+1 stored entries
  colptr = zeros(Int, k+2); rowval = zeros(Int, 2k+1)
  colptr[1] = 1
  for i = 1:k+1
    pos = colptr[i]
    if i ≤ k
      colptr[i+1] = pos + 2; rowval[pos] = i; rowval[pos+1] = i+1
    else
      colptr[i+1] = pos + 1; rowval[pos] = i
    end
  end
  colptr, rowval
end

function Krylov.hermitian_lanczos(A::B200CSR{T}, b::B200Vector{T}, k::Int;
                                  allow_breakdown::Bool=false, reorthogonalization::Bool=false) where T<:BlasT
  A.m == A.n || error("A must be square")
  length(b) == A.n || error("Inconsistent problem size")
  k ≥ 1 || error("k must be at least 1")
  V = B200Matrix{T}(undef, A.n, k+1)
  β = Ref{Cdouble}(0)
  nz = zeros(Cdouble, 3k-1)
  proc_check(ccall((:kb200_hermitian_lanczos, lib), Cint,
                   (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ref{Cdouble}, Ptr{Cdouble}, Cint),
                   ctx(), A.handle, k, dtype_id(T), b.ptr, V.ptr, β, nz, proc_flags(allow_breakdown, reorthogonalization)),
             "hermitian_lanczos")
  colptr, rowval = tridiagonal_pattern(k)
  return V, T(β[]), SparseMatrixCSC(k+1, k, colptr, rowval, T.(nz))
end

function Krylov.arnoldi(A::B200CSR{T}, b::B200Vector{T}, k::Int;
                        allow_breakdown::Bool=false, reorthogonalization::Bool=false) where T<:BlasT
  A.m == A.n || error("A must be square")
  length(b) == A.n || error("Inconsistent problem size")
  k ≥ 1 || error("k must be at least 1")
  V = B200Matrix{T}(undef, A.n, k+1)
  β = Ref{Cdouble}(0)
  H = zeros(Cdouble, k+1, k)
  proc_check(ccall((:kb200_arnoldi, lib), Cint,
                   (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ref{Cdouble}, Ptr{Cdouble}, Cint),
                   ctx(), A.handle, k, dtype_id(T), b.ptr, V.ptr, β, H, proc_flags(allow_breakdown, reorthogonalization)),
             "arnoldi")
  return V, T(β[]), T.(H)
end

function Krylov.golub_kahan(A::B200CSR{T}, b::B200Vector{T}, k::Int; allow_breakdown::Bool=false) where T<:BlasT
  length(b) == A.m || error("Inconsistent problem size")
  k ≥ 1 || error("k must be at least 1")
  V = B200Matrix{T}(undef, A.n, k+1)
  U = B200Matrix{T}(undef, A.m, k+1)
  β = Ref{Cdouble}(0)
  nz = zeros(Cdouble, 2k+1)
  proc_check(ccall((:kb200_golub_kahan, lib), Cint,
                   (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{Cdouble}, Ptr{Cdouble}, Cint),
                   ctx(), A.handle, C_NULL, k, dtype_id(T), b.ptr, V.ptr, U.ptr, β, nz, proc_flags(allow_breakdown)),
             "golub_kahan")
  colptr, rowval = bidiagonal_pattern(k)
  return V, U, T(β[]), SparseMatrixCSC(k+1, k+1, colptr, rowval, T.(nz))
end

function Krylov.nonhermitian_lanczos(A::B200CSR{T}, b::B200Vector{T}, c::B200Vector{T}, k::Int;
                                     allow_breakdown::Bool=false) where T<:BlasT
  A.m == A.n || error("A must be square")
  length(b) == length(c) == A.n || error("Inconsistent problem size")
  k ≥ 1 || error("k must be at least 1")
  V = B200Matrix{T}(undef, A.n, k+1)
  U = B200Matrix{T}(undef, A.n, k+1)
  β = Ref{Cdouble}(0); γ = Ref{Cdouble}(0)
  nzT = zeros(Cdouble, 3k-1); nzTᴴ = zeros(Cdouble, 3k-1)
  proc_check(ccall((:kb200_nonhermitian_lanczos, lib), Cint,
                   (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{Cdouble},
                    Ref{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint),
                   ctx(), A.handle, C_NULL, k, dtype_id(T), b.ptr, c.ptr, V.ptr, U.ptr, β, γ, nzT, nzTᴴ, proc_flags(allow_breakdown)),
             "nonhermitian_lanczos")
  colptr, rowval = tridiagonal_pattern(k)
  return V, T(β[]), SparseMatrixCSC(k+1, k, colptr, rowval, T.(nzT)), U, T(γ[]),
         SparseMatrixCSC(k+1, k, copy(colptr), copy(rowval), T.(nzTᴴ))
end

function Krylov.saunders_simon_yip(A::B200CSR{T}, b::B200Vector{T}, c::B200Vector{T}, k::Int;
                                   allow_breakdown::Bool=false) where T<:BlasT
  length(b) == A.m && length(c) == A.n || error("Inconsistent problem size")
  k ≥ 1 || error("k must be at least 1")
  V = B200Matrix{T}(undef, A.m, k+1)
  U = B200Matrix{T}(undef, A.n, k+1)
  β = Ref{Cdouble}(0); γ = Ref{Cdouble}(0)
  nzT = zeros(Cdouble, 3k-1); nzTᴴ = zeros(Cdouble, 3k-1)
  proc_check(ccall((:kb200_saunders_simon_yip, lib), Cint,
                   (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{Cdouble},
                    Ref{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint),
                   ctx(), A.handle, C_NULL, k, dtype_id(T), b.ptr, c.ptr, V.ptr, U.ptr, β, γ, nzT, nzTᴴ, proc_flags(allow_breakdown)),
             "saunders_simon_yip")
  colptr, rowval = tridiagonal_pattern(k)
  return V, T(β[]), SparseMatrixCSC(k+1, k, colptr, rowval, T.(nzT)), U, T(γ[]),
         SparseMatrixCSC(k+1, k, copy(colptr), copy(rowval), T.(nzTᴴ))
end

end # module
