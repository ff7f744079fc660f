# Package-extension shim for Clarabel.jl (see INTEGRATION.md).  Not executable in this repo's image
# (no Julia); kept in sync with INTEGRATION.md section 1.
module B200Ext
using Clarabel, SparseArrays
import Clarabel: AbstractDirectLDLSolver, ldlsolver_constructor, ldlsolver_matrix_shape,
                 ldlsolver_is_available, update_values!, scale_values!, refactor!, solve!,
                 linear_solver_info, LinearSolverInfo

const LIB = get(ENV, "CLARABEL_B200_LIB", "libclarabel_b200.so")

# mirrors `cb200_settings` in include/clarabel_b200.h (field order matters)
struct CB200Settings
    index_base::Int32; device::Int32
    static_regularization_enable::Int32
    static_regularization_constant::Float64; static_regularization_proportional::Float64
    dynamic_regularization_enable::Int32
    dynamic_regularization_eps::Float64; dynamic_regularization_delta::Float64
    iterative_refinement_enable::Int32
    iterative_refinement_reltol::Float64; iterative_refinement_abstol::Float64
    iterative_refinement_max_iter::Int32; iterative_refinement_stop_ratio::Float64
    ordering::Int32; amd_dense_scale::Float64; nd_leaf_size::Int32; use_cuda_graph::Int32
    reserved::NTuple{8,Int32}
end

mutable struct B200DirectLDLSolver{T} <: AbstractDirectLDLSolver{T}
    handle::Ptr{Cvoid}
    function B200DirectLDLSolver{T}(KKT::SparseMatrixCSC{T,Int64}, Dsigns::Vector{Int64}, settings) where {T}
        T === Float64 || error("B200 backend is Float64 only")
        cs = Ref{CB200Settings}()
        ccall((:cb200_default_settings, LIB), Cvoid, (Ref{CB200Settings},), cs)
        s = cs[]
        cs[] = CB200Settings(1, s.device,                     # index_base = 1: Julia indices
            settings.static_regularization_enable, settings.static_regularization_constant,
            settings.static_regularization_proportional, settings.dynamic_regularization_enable,
            settings.dynamic_regularization_eps, settings.dynamic_regularization_delta,
            settings.iterative_refinement_enable, settings.iterative_refinement_reltol,
            settings.iterative_refinement_abstol, settings.iterative_refinement_max_iter,
            settings.iterative_refinement_stop_ratio, s.ordering,   # 1 = auto: the LIBRARY picks the PSD-safe order when
            s.amd_dense_scale,                                       # K holds dense cone blocks (INTEGRATION.md section 5)
            s.nd_leaf_size, s.use_cuda_graph, s.reserved)
        h = Ref{Ptr{Cvoid}}(C_NULL)
        rc = ccall((:cb200_create, LIB), Int32,
                   (Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Int64}, Ref{CB200Settings}, Ref{Ptr{Cvoid}}),
                   size(KKT, 1), KKT.colptr, KKT.rowval, KKT.nzval, Dsigns, cs, h)
        rc == 0 || error("cb200_create: ", unsafe_string(ccall((:cb200_last_error, LIB), Cstring, ())))
        obj = new(h[])
        finalizer(o -> ccall((:cb200_destroy, LIB), Cvoid, (Ptr{Cvoid},), o.handle), obj)  # MOI.empty! finalizes the solver (MOI_wrapper.jl:133)
        return obj
    end
end

ldlsolver_constructor(::Val{:b200})  = B200DirectLDLSolver
ldlsolver_matrix_shape(::Val{:b200}) = :triu
ldlsolver_is_available(::Val{:b200}) = true

_chk(rc) = rc < 0 ? error(unsafe_string(ccall((:cb200_last_error, LIB), Cstring, ()))) : rc == 0

update_values!(s::B200DirectLDLSolver{T}, index::AbstractVector{Int64}, values::Vector{T}) where {T} =
    _chk(ccall((:cb200_update_values, LIB), Int32, (Ptr{Cvoid}, Ptr{Int64}, Ptr{Float64}, Int64),
               s.handle, index, values, length(index)))
scale_values!(s::B200DirectLDLSolver{T}, index::AbstractVector{Int64}, scale::T) where {T} =
    _chk(ccall((:cb200_scale_values, LIB), Int32, (Ptr{Cvoid}, Ptr{Int64}, Int64, Float64),
               s.handle, index, length(index), scale))
refactor!(s::B200DirectLDLSolver, K::SparseMatrixCSC) =                       # ::Bool, never throws on a bad pivot
    _chk(ccall((:cb200_refactor, LIB), Int32, (Ptr{Cvoid},), s.handle))
solve!(s::B200DirectLDLSolver{T}, K::SparseMatrixCSC{T}, x::Vector{T}, b::Vector{T}) where {T} =
    _chk(ccall((:cb200_solve, LIB), Int32, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}), s.handle, x, b))
function linear_solver_info(s::B200DirectLDLSolver)
    nnzA = Ref{Int64}(0); nnzL = Ref{Int64}(0); ng = Ref{Int32}(0)
    ccall((:cb200_info, LIB), Int32, (Ptr{Cvoid}, Ref{Int64}, Ref{Int64}, Ref{Int32}), s.handle, nnzA, nnzL, ng)
    LinearSolverInfo(:b200, ng[], true, nnzA[], nnzL[])
end

# update_scaling! of the symmetric cones on the device (INTEGRATION.md, "Cone scaling on the device").  `h` is a
# handle after cb200_set_maps; s, z have length m.  Returns ok_scale (false where update_scaling! returns false);
# afterwards cb200_update_cones(h, C_NULL, ..., C_NULL) refactors from the device state.
function b200_update_scaling!(h::Ptr{Cvoid}, s::Vector{Float64}, z::Vector{Float64})
    ok = Ref{Int32}(0)
    rc = ccall((:cb200_update_scaling, LIB), Int32, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ref{Int32}), h, s, z, ok)
    rc < 0 && error(unsafe_string(ccall((:cb200_last_error, LIB), Cstring, ())))
    return ok[] != 0
end
# The state for the host cone operations; pass C_NULL for what is not needed.  w, lam: m; eta, d: #SOC; u, v: the
# SOC rows; R, Rinv: sum of n^2 over the PSD cones (column-major, cone order); psd_lam: sum of n.
b200_get_scaling!(h::Ptr{Cvoid}, w, lam, eta, d, u, v, R, Rinv, psd_lam) =
    _chk(ccall((:cb200_get_scaling, LIB), Int32,
               (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
                Ptr{Float64}, Ptr{Float64}, Ptr{Float64}), h, w, lam, eta, d, u, v, R, Rinv, psd_lam))
end # module
