# B200PencilArrays.jl -- Julia veneer over libpa_b200 (include/pa_b200.h).
#
# NOT EXECUTED IN THIS REPOSITORY'S CI: the build image has no Julia (and no
# MPI).  The same C ABI is exercised call-for-call by the Python/ctypes host
# mirror and its tests; this file is the binding a PencilArrays.jl maintainer
# would load next to CUDA.jl.  It plugs in at the reference's own seam --
# multiple dispatch on the array type carried by the `Pencil`
# (Pencils.jl:282-304) -- in two ways:
#
#   (A) kernel level: the "generic array" methods of the hot path
#       copy_range!   (Transpositions.jl:568-583)  -> pa_box_copy (K1, no allocation)
#       _permutedims! (Transpositions.jl:648-664)  -> pa_box_copy (K2, ONE pass, no temp)
#       so that the reference's own transpose_send!/transpose_recv! loops and a
#       CUDA-aware MPI keep driving the exchange;
#   (B) whole path: transpose!(t::Transposition; waitall) (Transpositions.jl:170-179)
#       -> pa_transpose (pack / NCCL exchange / unpack pipelined on CUDA streams),
#       MPI.Waitall(t) -> pa_wait.
module B200PencilArrays

using PencilArrays
using PencilArrays: Pencils, Transpositions, MemoryOrder, LogicalOrder
using PencilArrays.Transpositions: Transposition, PointToPoint, Alltoallv, AbstractTransposeMethod
using StaticPermutations
using CUDA
import MPI

const libpa = get(ENV, "PA_B200_LIB", "libpa_b200.so")

# ---- status -> exception (pa_b200.h: pa_status) ------------------------------
function check(status::Cint)
    status == 0 && return nothing
    msg = unsafe_string(ccall((:pa_last_error, libpa), Cstring, ()))
    what = unsafe_string(ccall((:pa_strerror, libpa), Cstring, (Cint,), status))
    status in (1, 2) && throw(ArgumentError("$what: $msg"))       # PA_EINVAL, PA_EINCOMPAT
    status == 3 && throw(DimensionMismatch("$what: $msg"))        # PA_EDIM
    error("libpa_b200: $what: $msg")
end

stream_ptr() = reinterpret(Ptr{Cvoid}, CUDA.stream().handle)
devptr(x::CuArray) = reinterpret(Ptr{Cvoid}, pointer(x))

# ---- (A) kernel-level overrides ------------------------------------------------
# column-major strides (in elements) of dims
function colstrides(dims::NTuple{N,Int}) where {N}
    s = ones(Int64, N)
    for i in 2:N
        s[i] = s[i - 1] * dims[i - 1]
    end
    s
end

# pack: strided sub-box of the memory-order parent -> contiguous send/recv buffer
function Transpositions.copy_range!(
        dest::CuVector{T}, dest_offset::Integer,
        src::PencilArray{T,N,<:CuArray}, src_range_memorder::NTuple,
    ) where {T,N}
    src_p = parent(src)
    exdims = extra_dims(src)
    ranges = (src_range_memorder..., map(Base.OneTo, exdims)...)
    ext = Int64[length(r) for r in ranges]
    sstr = colstrides(size(src_p))
    dstr = colstrides(Tuple(ext))
    soff = sum((first(r) - 1) * s for (r, s) in zip(ranges, sstr))
    check(ccall((:pa_box_copy, libpa), Cint,
        (Cint, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
        length(ext), ext, sstr, dstr, sizeof(T),
        devptr(src_p) + soff * sizeof(T), devptr(dest) + dest_offset * sizeof(T),
        stream_ptr(), C_NULL))
    dest
end

# unpack: dense block (dims in Pi memory order) -> permuted sub-box of parent(dst),
# one pass, no temporary (the reference allocates `tmp` and copies twice, :659-661)
function Transpositions._permutedims!(
        ::Type{<:CuArray}, v::SubArray{T,N,<:CuArray}, src::CuArray{T,N}, perm,
    ) where {T,N}
    E = N - length(perm)
    pperm = Tuple(append(perm, Val(E)))          # v[k] = src[j], k[i] = j[pperm[i]]
    ext = Int64[size(src)...]
    sstr = colstrides(size(src))
    pstr = colstrides(size(parent(v)))
    dstr = zeros(Int64, N)
    for i in 1:N
        dstr[pperm[i]] = pstr[i]
    end
    doff = sum((first(r) - 1) * s for (r, s) in zip(parentindices(v), pstr))
    check(ccall((:pa_box_copy, libpa), Cint,
        (Cint, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
        N, ext, sstr, dstr, sizeof(T), devptr(src), devptr(parent(v)) + doff * sizeof(T),
        stream_ptr(), C_NULL))
    v
end

# ---- (B) whole-path override ------------------------------------------------------
mutable struct Handles
    topo::Ptr{Cvoid}
    pencils::IdDict{Any,Ptr{Cvoid}}
    plans::Dict{Any,Ptr{Cvoid}}
    comm::Ptr{Cvoid}
end
const HANDLES = IdDict{Any,Handles}()   # keyed by MPITopology (identity, like `!==` at :182)

function handles(topo)
    get!(HANDLES, topo) do
        dims = Int64[size(topo)...]
        rank = MPI.Comm_rank(get_comm(topo))
        h = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_topology_create, libpa), Cint, (Cint, Ptr{Int64}, Cint, Ptr{Ptr{Cvoid}}),
                    length(dims), dims, rank, h))
        # NCCL bootstrap over the MPI communicator the user already has
        id = zeros(UInt8, 128)
        rank == 0 && check(ccall((:pa_comm_unique_id, libpa), Cint, (Ptr{UInt8},), id))
        MPI.Bcast!(id, 0, get_comm(topo))
        c = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_set_device, libpa), Cint, (Cint,), CUDA.deviceid(CUDA.device())))
        check(ccall((:pa_comm_init_rank, libpa), Cint, (Ptr{UInt8}, Cint, Cint, Ptr{Ptr{Cvoid}}),
                    id, MPI.Comm_size(get_comm(topo)), rank, c))
        setup_flag_window!(c[], get_comm(topo))
        Handles(h[], IdDict{Any,Ptr{Cvoid}}(), Dict{Any,Ptr{Cvoid}}(), c[])
    end
end

# Flag window of the one-sided methods (pa_comm_flags_export / _import): every rank
# exports a few 64-bit words per source rank and maps everybody else's; window-open /
# window-close of PeerPut / PeerGet then ride inside the transfer kernel as NVLink
# signals.  Collective; if ANY rank fails, all keep the NCCL fences.
function setup_flag_window!(comm_handle::Ptr{Cvoid}, comm::MPI.Comm)
    rank, nranks = MPI.Comm_rank(comm), MPI.Comm_size(comm)
    handle = zeros(UInt8, 64)
    off = Ref{Int64}(0)
    ok = ccall((:pa_comm_flags_export, libpa), Cint, (Ptr{Cvoid}, Ptr{UInt8}, Ptr{Int64}),
               comm_handle, handle, off) == 0
    handles_all = MPI.Allgather(handle, comm)
    offs_all = MPI.Allgather([off[]], comm)
    ok = MPI.Allreduce(ok, &, comm)
    if ok
        for r in 0:(nranks - 1)
            r == rank && continue
            ok &= ccall((:pa_comm_flags_import, libpa), Cint, (Ptr{Cvoid}, Cint, Ptr{UInt8}, Int64),
                        comm_handle, r, view(handles_all, 64r+1:64r+64), offs_all[r + 1]) == 0
        end
    end
    MPI.Allreduce(ok, &, comm) ||
        check(ccall((:pa_set_tunable, libpa), Cint, (Cstring, Int64), "nccl_fences", 1))
    nothing
end

function pencil_handle(H::Handles, p::Pencil{N}) where {N}
    get!(H.pencils, p) do
        perm = permutation(p)
        permv = isidentity(perm) ? C_NULL : Cint[Tuple(perm)...]
        # pencils sharing send_buf (Pencils.jl:265-270) share the device arenas
        share = C_NULL
        for (q, hq) in H.pencils
            q.send_buf === p.send_buf && (share = hq; break)
        end
        h = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_pencil_create, libpa), Cint,
            (Ptr{Cvoid}, Cint, Ptr{Int64}, Ptr{Cint}, Ptr{Cint}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}),
            H.topo, N, Int64[size_global(p)...], Cint[decomposition(p)...], permv, share, h))
        h[]
    end
end

method_code(::PointToPoint) = Cint(0)
method_code(::Alltoallv) = Cint(1)

# GPU extensions (no reference counterpart): one-sided transposition methods.
# `PeerPut`: every remote block is stored by ONE kernel straight into the
# destination rank's `dest` over NVLink; `PeerGet`: pull flavour.  Usage:
#     t = Transposition(dest, src; method = B200PencilArrays.PeerPut())
#     B200PencilArrays.register_window!(t)      # collective, once per (dest | src) array
#     transpose!(t)
struct PeerPut <: AbstractTransposeMethod end
struct PeerGet <: AbstractTransposeMethod end
method_code(::PeerPut) = Cint(2)
method_code(::PeerGet) = Cint(3)

# Collective over the communicator, like MPI_Win_create: exchanges CUDA IPC
# handles of the window array (dest for PeerPut, src for PeerGet).
function register_window!(t::Transposition)
    plan, H = plan_handle(t)
    A = t.method isa PeerGet ? parent(t.Ai) : parent(t.Ao)
    register_window!(plan, A, t.Pi.topology, t.dim)
    t
end

# the same for a bare plan: `A` is the window array, R the grid dim of the exchange
function register_window!(plan::Ptr{Cvoid}, A, topo, R)
    comm = get_comm(topo)
    handle = zeros(UInt8, 64)
    off = Ref{Int64}(0)
    check(ccall((:pa_ipc_export, libpa), Cint, (Ptr{Cvoid}, Ptr{UInt8}, Ptr{Int64}), devptr(A), handle, off))
    handles_all = MPI.Allgather(handle, comm)            # 64 bytes per rank
    offs_all = MPI.Allgather([off[]], comm)
    R === nothing && return plan
    # ranks (in `comm`) of my grid line along R: topology.ranks maps Cartesian
    # coordinates to ranks (MPITopologies.jl:84-86,208-226); get_remote_indices (:539-549)
    coords = topo.coords_local
    line = [topo.ranks[ntuple(i -> i == R ? n : coords[i], length(coords))...] for n in 1:size(topo)[R]]
    me = MPI.Comm_rank(comm)
    for (n, r) in enumerate(line)
        r == me && continue
        mapped = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_ipc_import, libpa), Cint, (Ptr{UInt8}, Int64, Ptr{Ptr{Cvoid}}),
                    view(handles_all, 64r+1:64r+64), offs_all[r + 1], mapped))
        check(ccall((:pa_plan_set_window, libpa), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Cvoid}),
                    plan, devptr(A), n, mapped[]))
        # (each import holds a reference on the mapping: pair it with pa_ipc_release(handle)
        #  when the window array is freed)
    end
    plan
end

function plan_handle(t::Transposition{T}) where {T}
    H = handles(t.Pi.topology)
    ex = Int64[extra_dims(t.Ai)...]
    key = (objectid(t.Pi), objectid(t.Po), Tuple(ex), sizeof(T), method_code(t.method))
    plan = get!(H.plans, key) do
        h = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_plan_create, libpa), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cint, Ptr{Ptr{Cvoid}}),
            pencil_handle(H, t.Pi), pencil_handle(H, t.Po), length(ex), ex, sizeof(T),
            method_code(t.method), h))
        h[]
    end
    plan, H
end

const DeviceTransposition{T,N} = Transposition{T,N,<:Pencil,<:Pencil,
    <:PencilArray{T,N,<:CuArray},<:PencilArray{T,N,<:CuArray}}

# transpose!(t; waitall) (Transpositions.jl:170-179).
# `fft = :forward | :backward` (GPU extension, PA_FFT_FORWARD / PA_FFT_BACKWARD): the unpack
# and the 1-d FFT along dest's contiguous dimension -- the next step of a PencilFFTs plan --
# run as ONE kernel (ComplexF64, or ComplexF32 in single precision; power-of-two lines of
# 8..1024 points, staged methods or PeerGet -- there the kernel reads every line straight out
# of the peers' src arrays, with no staging; PeerPut is refused).
# PA_FFT_F32 for ComplexF32 elements: the plan only knows sizeof(T), and 8 bytes is Float64 too
fft_precision_flag(::Type{T}) where {T} = T === ComplexF32 ? Cuint(32) : Cuint(0)

function Transpositions.transpose!(t::DeviceTransposition{T}; waitall = true, fft = nothing) where {T}
    plan, H = plan_handle(t)
    flags = waitall ? Cuint(1) : Cuint(0)        # PA_WAITALL
    fft === :forward && (flags |= Cuint(8))
    fft === :backward && (flags |= Cuint(16))
    fft === nothing || (flags |= fft_precision_flag(T))   # PA_FFT_F32
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)   # a rank may own nothing (Pencils.jl:193-218)
    check(ccall((:pa_transpose, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, ptr_or_null(parent(t.Ai)), ptr_or_null(parent(t.Ao)), flags, stream_ptr()))
    t
end

# Whether `transpose!(t; fft)` can fuse the unpack and the FFT (pa_plan_fft_check_ex, in the
# precision of eltype).  The same answer on every rank of the grid line (global geometry only):
# choose the fused or the separate transpose + transform up front.
fft_fusable(t::DeviceTransposition{T}) where {T} =
    ccall((:pa_plan_fft_check_ex, libpa), Cint, (Ptr{Cvoid}, Cuint), first(plan_handle(t)),
          fft_precision_flag(T)) == 0

# In-place 1-d FFT of `u` along its contiguous dimension (same kernel, no transposition): with
# the two fused transposes this is a whole PencilFFTs-style 3-d transform in three kernels.
# ComplexF64 or ComplexF32 (the flag follows eltype through transpose!).
fft_lines!(u::PencilArray{T,N,<:CuArray}; direction = :forward) where {T,N} =
    (Transpositions.transpose!(Transposition(u, u); fft = direction); u)

# Real-to-complex 1-d FFT along the first memory dimension (not decomposed), step 1 of a
# PencilFFTs real-input plan: `dest = rfft(src)` there.  `src` lives on a pencil of global size
# (..., N, ...), `dest` on `Pencil(pencil(src); size_global = (..., N÷2+1, ...))`; N a power of
# two in 16..2048.  `brfft!` is the unnormalised inverse (AbstractFFTs' `brfft`); it ignores the
# imaginary parts of bins 1 and N÷2+1 and leaves `src` unmodified.  One kernel, no communication.
# Float64 <-> ComplexF64, or Float32 <-> ComplexF32 in single precision (PA_FFT_F32).
function _rfft!(real::PencilArray{R,N,<:CuArray}, cplx::PencilArray{Complex{R},N,<:CuArray},
                flags::Cuint, src, dst) where {R<:Union{Float64,Float32},N}
    R === Float32 && (flags |= Cuint(32))        # PA_FFT_F32
    H = handles(pencil(real).topology)
    extra_dims(real) == extra_dims(cplx) ||
        throw(ArgumentError("incompatible extra dimensions: $(extra_dims(real)) != $(extra_dims(cplx))"))
    ex = Int64[extra_dims(real)...]
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_rfft, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Int64}, Cuint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
        pencil_handle(H, pencil(real)), pencil_handle(H, pencil(cplx)), length(ex), ex, flags,
        ptr_or_null(parent(src)), ptr_or_null(parent(dst)), stream_ptr()))
end

rfft!(dest::PencilArray{ComplexF64,N,<:CuArray}, src::PencilArray{Float64,N,<:CuArray}) where {N} =
    (_rfft!(src, dest, Cuint(8), src, dest); dest)       # PA_FFT_FORWARD
brfft!(dest::PencilArray{Float64,N,<:CuArray}, src::PencilArray{ComplexF64,N,<:CuArray}) where {N} =
    (_rfft!(dest, src, Cuint(16), src, dest); dest)      # PA_FFT_BACKWARD
rfft!(dest::PencilArray{ComplexF32,N,<:CuArray}, src::PencilArray{Float32,N,<:CuArray}) where {N} =
    (_rfft!(src, dest, Cuint(8), src, dest); dest)       # PA_FFT_FORWARD | PA_FFT_F32
brfft!(dest::PencilArray{Float32,N,<:CuArray}, src::PencilArray{ComplexF32,N,<:CuArray}) where {N} =
    (_rfft!(dest, src, Cuint(16), src, dest); dest)      # PA_FFT_BACKWARD | PA_FFT_F32

# Real-to-real 1-d transform along the first memory dimension (not decomposed), PencilFFTs'
# Transforms.R2R with FFTW's unnormalised kinds: `kind` is FFTW.REDFT10 (DCT-II), REDFT01
# (DCT-III), RODFT10 (DST-II) or RODFT01 (DST-III) -- the constants pass straight through (4, 5,
# 8, 9).  `dest` and `src` share the pencil geometry and extra dims; `dest === src` runs in
# place.  N a power of two in 16..2048.  One kernel, no communication.
function r2r!(dest::PencilArray{R,N,<:CuArray}, src::PencilArray{R,N,<:CuArray},
              kind::Integer) where {R<:Union{Float64,Float32},N}
    pd, ps = pencil(dest), pencil(src)
    (pd === ps || (topology(pd) === topology(ps) && size_global(pd) == size_global(ps) &&
                   decomposition(pd) == decomposition(ps) && permutation(pd) == permutation(ps))) ||
        throw(ArgumentError("r2r!: the arrays must have the same pencil geometry"))
    extra_dims(dest) == extra_dims(src) ||
        throw(ArgumentError("incompatible extra dimensions: $(extra_dims(dest)) != $(extra_dims(src))"))
    H = handles(topology(pd))
    ex = Int64[extra_dims(dest)...]
    flags = R === Float32 ? Cuint(32) : Cuint(0)   # PA_FFT_F32
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_r2r, libpa), Cint,
        (Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cuint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
        pencil_handle(H, pd), length(ex), ex, Cint(kind), flags,
        ptr_or_null(parent(src)), ptr_or_null(parent(dest)), stream_ptr()))
    dest
end

# Fused y->x transpose + complex-to-real transform (pa_transpose_brfft): the last step of a
# PencilFFTs real-input backward transform in one kernel per GPU after the exchange, `dest =
# brfft(transpose(src))`, without the complex x-pencil array.  `src`: Complex{R} on the complex
# y-pencil; `dest`: R on the real x-pencil; `pc`: the complex x-pencil the plan transposes to,
# `Pencil(pencil(dest); size_global = (..., N÷2+1, ...))` -- passed explicitly because a Julia
# `Transposition` holds arrays of one element type.  PointToPoint or Alltoallv.
function brfft_plan(src::PencilArray{Complex{R}}, pc::Pencil, method) where {R}
    H = handles(pencil(src).topology)
    ex = Int64[extra_dims(src)...]
    key = (objectid(pencil(src)), objectid(pc), Tuple(ex), sizeof(Complex{R}), method_code(method))
    plan = get!(H.plans, key) do
        h = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_plan_create, libpa), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cint, Ptr{Ptr{Cvoid}}),
            pencil_handle(H, pencil(src)), pencil_handle(H, pc), length(ex), ex, sizeof(Complex{R}),
            method_code(method), h))
        h[]
    end
    plan, H
end

function transpose_brfft!(dest::PencilArray{R,N,<:CuArray}, src::PencilArray{Complex{R},N,<:CuArray},
                          pc::Pencil; method = PointToPoint(), waitall = true) where {R<:Union{Float64,Float32},N}
    plan, H = brfft_plan(src, pc, method)
    flags = (waitall ? Cuint(1) : Cuint(0)) | fft_precision_flag(Complex{R})   # PA_WAITALL, PA_FFT_F32
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_transpose_brfft, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, pencil_handle(H, pencil(dest)), ptr_or_null(parent(src)), ptr_or_null(parent(dest)),
        flags, stream_ptr()))
    dest
end

# Whether transpose_brfft! can run on this geometry (pa_plan_brfft_check): the same answer on
# every rank of the grid line.
brfft_fusable(src::PencilArray{Complex{R}}, pc::Pencil; method = PointToPoint()) where {R} =
    ccall((:pa_plan_brfft_check, libpa), Cint, (Ptr{Cvoid}, Cuint), first(brfft_plan(src, pc, method)),
          fft_precision_flag(Complex{R})) == 0

# Fused transposition of real arrays + a line transform along dest's first memory dimension, in
# one kernel per GPU after the exchange (pa_transpose_r2r / pa_transpose_rfft): the steps of a
# wall-bounded PencilFFTs transform without the real array in between.
#   transpose_r2r!(dest, src, kind): dest = r2r(transpose(src), kind), both R on real pencils;
#     kind FFTW.REDFT10 / REDFT01 / RODFT10 / RODFT01 as in r2r!.
#   transpose_rfft!(dest, src, pr): dest = rfft(transpose(src)), `src` R on the real x-pencil,
#     `dest` Complex{R} on the complex y-pencil; `pr`: the real y-pencil the plan transposes to,
#     `Pencil(pencil(dest); size_global = (..., N, ...))` -- passed explicitly, as in
#     transpose_brfft!.
# Byte for byte the unfused pairs.  PointToPoint or Alltoallv; N a power of two in 16..2048.
function real_plan(src::PencilArray{R}, pr::Pencil, method) where {R<:Union{Float64,Float32}}
    H = handles(pencil(src).topology)
    ex = Int64[extra_dims(src)...]
    key = (objectid(pencil(src)), objectid(pr), Tuple(ex), sizeof(R), method_code(method))
    plan = get!(H.plans, key) do
        h = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_plan_create, libpa), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cint, Ptr{Ptr{Cvoid}}),
            pencil_handle(H, pencil(src)), pencil_handle(H, pr), length(ex), ex, sizeof(R),
            method_code(method), h))
        h[]
    end
    plan, H
end

function transpose_r2r!(dest::PencilArray{R,N,<:CuArray}, src::PencilArray{R,N,<:CuArray},
                        kind::Integer; method = PointToPoint(), waitall = true) where {R<:Union{Float64,Float32},N}
    plan, H = real_plan(src, pencil(dest), method)
    flags = (waitall ? Cuint(1) : Cuint(0)) | (R === Float32 ? Cuint(32) : Cuint(0))   # PA_WAITALL, PA_FFT_F32
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_transpose_r2r, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, Cint(kind), ptr_or_null(parent(src)), ptr_or_null(parent(dest)), flags, stream_ptr()))
    dest
end

function transpose_rfft!(dest::PencilArray{Complex{R},N,<:CuArray}, src::PencilArray{R,N,<:CuArray},
                         pr::Pencil; method = PointToPoint(), waitall = true) where {R<:Union{Float64,Float32},N}
    plan, H = real_plan(src, pr, method)
    flags = (waitall ? Cuint(1) : Cuint(0)) | (R === Float32 ? Cuint(32) : Cuint(0))   # PA_WAITALL, PA_FFT_F32
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_transpose_rfft, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, pencil_handle(H, pencil(dest)), ptr_or_null(parent(src)), ptr_or_null(parent(dest)),
        flags, stream_ptr()))
    dest
end

# Whether transpose_r2r! / transpose_rfft! can run on this geometry (pa_plan_real_check, one
# answer for both): the same answer on every rank of the grid line.
real_fusable(src::PencilArray{R}, pr::Pencil; method = PointToPoint()) where {R<:Union{Float64,Float32}} =
    ccall((:pa_plan_real_check, libpa), Cint, (Ptr{Cvoid}, Cuint), first(real_plan(src, pr, method)),
          R === Float32 ? Cuint(32) : Cuint(0)) == 0

# ---- host arrays: a chain of transpositions on `Array`-backed data ------------------
# pa_host_chain_*: one submit = upload, every transpose! on the device, download;
# asynchronous, double-buffered (download of one submit || upload of the next).
mutable struct HostChain
    h::Ptr{Cvoid}
end
function HostChain(ts::Vector{<:Transposition})
    plans = Ptr{Cvoid}[plan_handle(t)[1] for t in ts]
    H = handles(first(ts).Pi.topology)
    h = Ref{Ptr{Cvoid}}()
    check(ccall((:pa_host_chain_create, libpa), Cint, (Cint, Ptr{Ptr{Cvoid}}, Ptr{Cvoid}, Ptr{Ptr{Cvoid}}),
                length(plans), plans, H.comm, h))
    finalizer(c -> ccall((:pa_host_chain_destroy, libpa), Cvoid, (Ptr{Cvoid},), c.h), HostChain(h[]))
end
function submit!(c::HostChain, host_dst::Array, host_src::Array)   # pin both with CUDA.pin
    k = Ref{Int64}(0)
    check(ccall((:pa_host_chain_submit, libpa), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Int64}),
                c.h, pointer(host_src), pointer(host_dst), k))
    k[]
end
Base.wait(c::HostChain, ticket = -1) =
    check(ccall((:pa_host_chain_wait, libpa), Cint, (Ptr{Cvoid}, Int64), c.h, ticket))

# ---- PencilIO: MPIIODriver files straight from / into device arrays ------------------
# The reference's set_view! + MPI.File.write_all (mpi_io.jl:338-380) needs host memory;
# these methods keep its file format (and its own add_metadata / JSON sidecar) and move
# the rank's sub-box with pa_io_write / pa_io_read.
using PencilArrays.PencilIO: PencilIO
function PencilIO.write_discontiguous(ff::MPI.FileHandle, x::PencilArray{T,N,<:CuArray};
                                      offset, collective, filename, infokws...) where {T,N}
    H = handles(topology(pencil(x)))
    ex = Int64[extra_dims(x)...]
    check(ccall((:pa_io_write, libpa), Cint,
        (Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cint, Ptr{Cvoid}, Cstring, Int64),
        pencil_handle(H, pencil(x)), length(ex), ex, sizeof(T), 0, devptr(parent(x)), filename, offset))
    nothing
end
function PencilIO.read_discontiguous!(ff::MPI.FileHandle, x::PencilArray{T,N,<:CuArray};
                                      offset, collective, filename, infokws...) where {T,N}
    H = handles(topology(pencil(x)))
    ex = Int64[extra_dims(x)...]
    check(ccall((:pa_io_read, libpa), Cint,
        (Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cint, Ptr{Cvoid}, Cstring, Int64),
        pencil_handle(H, pencil(x)), length(ex), ex, sizeof(T), 0, devptr(parent(x)), filename, offset))
    x
end
# (the chunks = true pair, write_contiguous / read_contiguous!, passes 1 instead of 0; the
#  caller supplies `filename = get_filename(file)` -- two one-line forwarding methods of
#  setindex!(::MPIFile, …) / _read_mpiio! in the extension)

# MPI.Waitall(t) (Transpositions.jl:127-130)
function MPI.Waitall(t::DeviceTransposition)
    plan, _ = plan_handle(t)
    check(ccall((:pa_wait, libpa), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), plan, stream_ptr()))
    nothing
end

# Send-side fused transform + transposition (pa_fft_put / pa_rfft_put): the transform along the
# FIRST memory dimension of `src` (not decomposed) runs in the put kernel -- one kernel per GPU
# loads every local source line, transforms it and stores the bins into the peers' dest through
# the PeerPut window.  PeerPut, or a local transposition with any method; byte for byte the
# unfused pair (fft_lines! on a copy / rfft!, then transpose!).
#   fft_transpose!(t; direction = :forward | :backward): dest = transpose(fft(src)) on a complex
#     Transposition (register_window! it first under PeerPut, as for transpose!).
#   rfft_transpose!(dest, src, pc): dest = transpose(rfft(src)), `src` R on the real x-pencil,
#     `dest` Complex{R} on the complex y-pencil; `pc`: the complex x-pencil the plan transposes
#     from, `Pencil(pencil(src); size_global = (..., N÷2+1, ...))` -- passed explicitly, as in
#     transpose_brfft!.  Under PeerPut it registers dest's window itself (collective).
function fft_transpose!(t::DeviceTransposition{T}; direction = :forward, waitall = true) where {T}
    plan, H = plan_handle(t)
    dir = direction === :forward ? Cuint(8) : direction === :backward ? Cuint(16) :
        throw(ArgumentError("direction must be :forward or :backward"))
    flags = (waitall ? Cuint(1) : Cuint(0)) | dir | fft_precision_flag(T)   # PA_WAITALL, PA_FFT_*
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_fft_put, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, ptr_or_null(parent(t.Ai)), ptr_or_null(parent(t.Ao)), flags, stream_ptr()))
    t
end

function rfft_put_plan(pc::Pencil, dest::PencilArray{Complex{R}}, method) where {R}
    H = handles(pc.topology)
    ex = Int64[extra_dims(dest)...]
    key = (objectid(pc), objectid(pencil(dest)), Tuple(ex), sizeof(Complex{R}), method_code(method))
    plan = get!(H.plans, key) do
        h = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_plan_create, libpa), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cint, Ptr{Ptr{Cvoid}}),
            pencil_handle(H, pc), pencil_handle(H, pencil(dest)), length(ex), ex, sizeof(Complex{R}),
            method_code(method), h))
        h[]
    end
    plan, H
end

function rfft_transpose!(dest::PencilArray{Complex{R},N,<:CuArray}, src::PencilArray{R,N,<:CuArray},
                         pc::Pencil; method = PeerPut(), waitall = true) where {R<:Union{Float64,Float32},N}
    plan, H = rfft_put_plan(pc, dest, method)
    flag = R === Float32 ? Cuint(32) : Cuint(0)   # PA_FFT_F32
    # refused (on every rank of the line alike) before the collective window setup
    check(ccall((:pa_plan_rfft_put_check, libpa), Cint, (Ptr{Cvoid}, Cuint), plan, flag))
    if method isa PeerPut
        R_dim = findfirst(i -> decomposition(pc)[i] != decomposition(pencil(dest))[i],
                          1:length(decomposition(pc)))
        register_window!(plan, parent(dest), pc.topology, R_dim)
    end
    flags = (waitall ? Cuint(1) : Cuint(0)) | flag   # PA_WAITALL
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_rfft_put, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, pencil_handle(H, pencil(src)), ptr_or_null(parent(src)), ptr_or_null(parent(dest)),
        flags, stream_ptr()))
    dest
end

# Whether fft_transpose! / rfft_transpose! can run (pa_plan_fft_put_check / pa_plan_rfft_put_check):
# the same answer on every rank of the grid line.
fft_first_fusable(t::DeviceTransposition{T}) where {T} =
    ccall((:pa_plan_fft_put_check, libpa), Cint, (Ptr{Cvoid}, Cuint), first(plan_handle(t)),
          fft_precision_flag(T)) == 0
rfft_first_fusable(dest::PencilArray{Complex{R}}, pc::Pencil; method = PeerPut()) where {R} =
    ccall((:pa_plan_rfft_put_check, libpa), Cint, (Ptr{Cvoid}, Cuint), first(rfft_put_plan(pc, dest, method)),
          R === Float32 ? Cuint(32) : Cuint(0)) == 0

# The wall-bounded legs of the send-side fusion (pa_r2r_put / pa_brfft_put, DESIGN §3j), on REAL
# plans: N reals per line along the first memory dimension of the plan's input pencil.  PeerPut, or
# a local transposition with any method; byte for byte the unfused pair.  Under PeerPut they
# register dest's window themselves (collective), after the verdict -- refused on every rank of the
# line alike before any window setup.
#   r2r_transpose!(dest, src, kind): dest = transpose(r2r(src, kind)), `src` and `dest` R on two real
#     pencils, `kind` one of REDFT10 / REDFT01 / RODFT10 / RODFT01.
#   brfft_transpose!(dest, src, pr): dest = transpose(brfft(src)), `src` Complex{R} on the complex
#     y-pencil, `dest` R on the real x-pencil; `pr`: the real y-pencil the plan transposes from,
#     `Pencil(pencil(src); size_global = (..., N, ...))` -- passed explicitly, as in
#     rfft_transpose!.
function real_put_plan(pr::Pencil, dest::PencilArray{R}, method) where {R<:Union{Float64,Float32}}
    H = handles(pr.topology)
    ex = Int64[extra_dims(dest)...]
    key = (objectid(pr), objectid(pencil(dest)), Tuple(ex), sizeof(R), method_code(method))
    plan = get!(H.plans, key) do
        h = Ref{Ptr{Cvoid}}()
        check(ccall((:pa_plan_create, libpa), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Int64}, Cint, Cint, Ptr{Ptr{Cvoid}}),
            pencil_handle(H, pr), pencil_handle(H, pencil(dest)), length(ex), ex, sizeof(R),
            method_code(method), h))
        h[]
    end
    plan, H
end

function real_put_window!(plan, pr::Pencil, dest::PencilArray, method, flag)
    check(ccall((:pa_plan_real_put_check, libpa), Cint, (Ptr{Cvoid}, Cuint), plan, flag))
    if method isa PeerPut
        R_dim = findfirst(i -> decomposition(pr)[i] != decomposition(pencil(dest))[i],
                          1:length(decomposition(pr)))
        R_dim === nothing || register_window!(plan, parent(dest), pr.topology, R_dim)
    end
end

function r2r_transpose!(dest::PencilArray{R,N,<:CuArray}, src::PencilArray{R,N,<:CuArray}, kind::Integer;
                        method = PeerPut(), waitall = true) where {R<:Union{Float64,Float32},N}
    plan, H = real_put_plan(pencil(src), dest, method)
    flag = R === Float32 ? Cuint(32) : Cuint(0)   # PA_FFT_F32
    real_put_window!(plan, pencil(src), dest, method, flag)
    flags = (waitall ? Cuint(1) : Cuint(0)) | flag   # PA_WAITALL
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_r2r_put, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, Cint(kind), ptr_or_null(parent(src)), ptr_or_null(parent(dest)), flags, stream_ptr()))
    dest
end

function brfft_transpose!(dest::PencilArray{R,N,<:CuArray}, src::PencilArray{Complex{R},N,<:CuArray},
                          pr::Pencil; method = PeerPut(), waitall = true) where {R<:Union{Float64,Float32},N}
    plan, H = real_put_plan(pr, dest, method)
    flag = R === Float32 ? Cuint(32) : Cuint(0)   # PA_FFT_F32
    real_put_window!(plan, pr, dest, method, flag)
    flags = (waitall ? Cuint(1) : Cuint(0)) | flag   # PA_WAITALL
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    check(ccall((:pa_brfft_put, libpa), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Cuint, Ptr{Cvoid}),
        plan, H.comm, pencil_handle(H, pencil(src)), ptr_or_null(parent(src)), ptr_or_null(parent(dest)),
        flags, stream_ptr()))
    dest
end

# Whether r2r_transpose! / brfft_transpose! can run (pa_plan_real_put_check, one answer for both):
# the same answer on every rank of the grid line.
real_first_fusable(dest::PencilArray{R}, pr::Pencil; method = PeerPut()) where {R<:Union{Float64,Float32}} =
    ccall((:pa_plan_real_put_check, libpa), Cint, (Ptr{Cvoid}, Cuint), first(real_put_plan(pr, dest, method)),
          R === Float32 ? Cuint(32) : Cuint(0)) == 0

# ---- global reductions (reductions.jl:10-38) ------------------------------------------------------
# mapreduce / sum / maximum / minimum / any / all of CuArray-backed PencilArrays with the functions
# pa_reduce recognises run as ONE kernel per rank (local pass + combine through the flag window);
# the result is read back as a scalar, as the reference's MPI.Allreduce returns one.  Any other
# function falls back to the reference's generic method (local mapreduce + MPI.Allreduce).
const PA_DTYPE = IdDict{Type,Cint}(Float64 => 0, Float32 => 1, ComplexF64 => 2, ComplexF32 => 3,
                                   Int32 => 4, Int64 => 5)
const PA_RESULT = Dict{Cint,Type}(0 => Float64, 1 => Float32, 2 => ComplexF64, 3 => ComplexF32,
                                  4 => Int32, 5 => Int64, 6 => Bool)
realdot(x, y) = real(x * conj(y))
pa_map(::typeof(identity)) = Cint(0)
pa_map(::typeof(abs)) = Cint(1)
pa_map(::typeof(abs2)) = Cint(2)
pa_map(::typeof(realdot)) = Cint(3)
pa_map(::Any) = nothing
pa_op(::typeof(+)) = Cint(0)
pa_op(::typeof(Base.add_sum)) = Cint(0)
pa_op(::typeof(max)) = Cint(1)
pa_op(::typeof(min)) = Cint(2)
pa_op(::Any) = nothing
# predicates: Base.Fix2 of a comparison (==(2), >(0), ...) or isnan / isfinite
pa_pred(f::Base.Fix2{typeof(==)}) = (Cint(1) << 4, f.x)
pa_pred(f::Base.Fix2{typeof(!=)}) = (Cint(2) << 4, f.x)
pa_pred(f::Base.Fix2{typeof(<)}) = (Cint(3) << 4, f.x)
pa_pred(f::Base.Fix2{typeof(<=)}) = (Cint(4) << 4, f.x)
pa_pred(f::Base.Fix2{typeof(>)}) = (Cint(5) << 4, f.x)
pa_pred(f::Base.Fix2{typeof(>=)}) = (Cint(6) << 4, f.x)
pa_pred(::typeof(isnan)) = (Cint(7) << 4, nothing)
pa_pred(::typeof(isfinite)) = (Cint(8) << 4, nothing)
pa_pred(::Any) = nothing

const CuPencilArray{T,N} = PencilArray{T,N,<:CuArray}

function pa_reduce(u::CuPencilArray{T}, v, map::Cint, op::Cint, value) where {T}
    v === nothing || PencilArrays._check_compatible_arrays(u, v)
    H = handles(topology(pencil(u)))
    dt = PA_DTYPE[T]
    rt = Ref{Cint}()
    check(ccall((:pa_reduce_result_type, libpa), Cint, (Cint, Cint, Cint, Ptr{Cint}), dt, map, op, rt))
    R = PA_RESULT[rt[]]
    result = CuArray{R}(undef, 1)
    VT = map == 0 ? T : real(T)
    ref = value === nothing ? C_NULL : Ref{VT}(convert(VT, value))
    ex = Int64[extra_dims(u)...]
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    GC.@preserve ref check(ccall((:pa_reduce, libpa), Cint,
        (Ptr{Cvoid}, Cint, Ptr{Int64}, Ptr{Cvoid}, Cint, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid},
         Ptr{Cvoid}, Ptr{Cvoid}),
        pencil_handle(H, pencil(u)), length(ex), ex, H.comm, dt, map, op,
        ref === C_NULL ? C_NULL : Base.unsafe_convert(Ptr{Cvoid}, ref), ptr_or_null(parent(u)),
        v === nothing ? C_NULL : ptr_or_null(parent(v)), devptr(result), stream_ptr()))
    CUDA.@allowscalar result[1]
end

const PA_ELTYPES = Union{Float64,Float32,ComplexF64,ComplexF32,Int32,Int64}

function Base.mapreduce(f::F, op::OP, u::CuPencilArray{T}, etc::Vararg{CuPencilArray{T}};
                        kws...) where {F,OP,T<:PA_ELTYPES}
    m, o = pa_map(f), pa_op(op)
    nargs = 1 + length(etc)
    if isempty(kws) && m !== nothing && o !== nothing && (nargs == 2) == (m == 3) && nargs <= 2
        return pa_reduce(u, nargs == 2 ? etc[1] : nothing, m, o, nothing)
    end
    # the reference's generic method (reductions.jl:10-18)
    foreach(v -> PencilArrays._check_compatible_arrays(u, v), etc)
    rlocal = mapreduce(f, op, map(parent, (u, etc...))...; kws...)
    MPI.Allreduce(rlocal, MPI.Op(op, typeof(rlocal); iscommutative = true), get_comm(u))
end

Base.sum(f::F, u::CuPencilArray{<:PA_ELTYPES}) where {F} = mapreduce(f, Base.add_sum, u)
Base.sum(u::CuPencilArray{<:PA_ELTYPES}) = mapreduce(identity, Base.add_sum, u)
Base.maximum(f::F, u::CuPencilArray{<:PA_ELTYPES}) where {F} = mapreduce(f, max, u)
Base.maximum(u::CuPencilArray{<:PA_ELTYPES}) = mapreduce(identity, max, u)
Base.minimum(f::F, u::CuPencilArray{<:PA_ELTYPES}) where {F} = mapreduce(f, min, u)
Base.minimum(u::CuPencilArray{<:PA_ELTYPES}) = mapreduce(identity, min, u)

# The kernel compares in the element type; Julia compares in the promoted type.  The two agree
# only when the value converts exactly (0.1 against Float32 data does not: 0.1f0 > 0.1).
function exact_in(::Type{T}, x) where {T}
    x isa Number || return false
    y = try
        convert(T, x)
    catch
        return false
    end
    return y == x || (isnan(y) && isnan(x))
end

for (fn, code) in ((:any, 3), (:all, 4))
    @eval function Base.$fn(f::F, u::CuPencilArray{T}) where {F<:Function,T<:PA_ELTYPES}
        p = pa_pred(f)
        if p === nothing || !(p[2] === nothing || exact_in(T, p[2]))
            # the reference's generic method (reductions.jl:30-38)
            xlocal = $fn(f, parent(u))::Bool
            return MPI.Allreduce(xlocal, $(fn === :any ? :| : :&), get_comm(u))
        end
        pa_reduce(u, nothing, Cint(0), Cint($code) | p[1], p[2])::Bool
    end
end

# ---- reductions along dims (pa_reduce_dims, DESIGN §3l) -----------------------------------------
# mapreduce_dims(f, op, u[, v]; dims): `dims` are LOGICAL dims (1..N spatial, N+1.. extra, as
# ndims(u) counts them).  Returns this rank's CuArray, laid out like parent(u) with extent 1 along
# the reduced dims: the reduction over their global ranges at this rank's kept indices, combined
# over the ranks that share them.  Base.mapreduce(...; dims) keeps the reference's method, which
# counts memory-order dims and Allreduces over all ranks (right only when every decomposed dim is
# reduced).  For any / all pass op = any or all and f = a predicate pa_pred recognises.
function mapreduce_dims(f::F, op::OP, u::CuPencilArray{T}, etc::Vararg{CuPencilArray{T}};
                        dims) where {F,OP,T<:PA_ELTYPES}
    length(etc) <= 1 || throw(ArgumentError("mapreduce_dims takes one or two arrays"))
    v = isempty(etc) ? nothing : etc[1]
    v === nothing || PencilArrays._check_compatible_arrays(u, v)
    if op === any || op === all
        p = pa_pred(f)
        (p !== nothing && (p[2] === nothing || exact_in(T, p[2]))) ||
            throw(ArgumentError("mapreduce_dims: predicate $f is not one the library runs"))
        map, code, value = Cint(0), Cint(op === any ? 3 : 4) | p[1], p[2]
    else
        map, code, value = pa_map(f), pa_op(op), nothing
        (map !== nothing && code !== nothing && (v !== nothing) == (map == 3)) ||
            throw(ArgumentError("mapreduce_dims: ($f, $op) is not a reduction the library runs"))
    end
    H = handles(topology(pencil(u)))
    dt = PA_DTYPE[T]
    rt = Ref{Cint}()
    check(ccall((:pa_reduce_result_type, libpa), Cint, (Cint, Cint, Cint, Ptr{Cint}), dt, map, code, rt))
    ds = Cint[d for d in dims]
    N = ndims(pencil(u))
    pp = permutation(pencil(u))
    perm = isidentity(pp) ? Tuple(1:N) : Tuple(pp)  # memory dim m holds logical dim perm[m]
    shape = collect(size(parent(u)))
    for d in ds
        1 <= d <= length(shape) || throw(ArgumentError("dim $d out of range 1..$(length(shape))"))
        shape[d <= N ? findfirst(==(d), perm) : d] = 1
    end
    result = CuArray{PA_RESULT[rt[]]}(undef, shape...)
    VT = map == 0 ? T : real(T)
    ref = value === nothing ? C_NULL : Ref{VT}(convert(VT, value))
    ex = Int64[extra_dims(u)...]
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    GC.@preserve ref ds check(ccall((:pa_reduce_dims, libpa), Cint,
        (Ptr{Cvoid}, Cint, Ptr{Int64}, Ptr{Cvoid}, Cint, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid},
         Cint, Ptr{Cint}, Ptr{Cvoid}, Ptr{Cvoid}),
        pencil_handle(H, pencil(u)), length(ex), ex, H.comm, dt, map, code,
        ref === C_NULL ? C_NULL : Base.unsafe_convert(Ptr{Cvoid}, ref), ptr_or_null(parent(u)),
        v === nothing ? C_NULL : ptr_or_null(parent(v)), length(ds), ds, ptr_or_null(result),
        stream_ptr()))
    result
end

# ---- shell-binned spectra (pa_shell_spectrum, DESIGN §3m) ----------------------------------------
# shell_spectrum(abs2, û; ...) and shell_spectrum(realdot, û, v̂; ...): E(b) = Σ over the modes
# with bin(|k|) == b of w · abs2(û) (or w · real(û · conj(v̂))), the global spectrum as a CuVector
# of nbins values (Float64, or Float32 for ComplexF32 arrays), the same bits on every rank.
# rfft_dim: the logical dim holding the n ÷ 2 + 1 bins of a real-to-complex transform of length
# rfft_n (default 2 (M - 1)); scales: one per spatial dim (2π / L_d; default 1); width: the shell
# width; nbins: default the bin of the extreme mode plus one (pa_shell_spectrum_nbins).
# dims / keep (pa_shell_spectrum_dims, DESIGN §3n): |k| over the bin dims `dims` only (spatial,
# default all), the logical dims in `keep` (extra dims N+1.. included) kept, every other dim summed:
# dims = (1, 3), keep = (2,) is E(k_h; y).  With `keep` the result has size(parent(u)) with every
# non-kept position 1 and a leading nbins dim (bins fastest, as the C layout result[b + nbins * o]),
# this rank's local range along each kept dim.
function shell_spectrum(f::F, u::CuPencilArray{T}, etc::Vararg{CuPencilArray{T}};
                        rfft_dim::Integer = 0, rfft_n::Integer = 0, scales = nothing,
                        width::Real = 1.0, nbins = nothing, dims = nothing,
                        keep = ()) where {F,T<:Union{ComplexF64,ComplexF32}}
    (dims === nothing && isempty(keep)) ||
        return shell_spectrum_dims(f, u, etc...; rfft_dim, rfft_n, scales, width, nbins,
                                   dims = dims === nothing ? Tuple(1:ndims(pencil(u))) : dims, keep)
    length(etc) <= 1 || throw(ArgumentError("shell_spectrum takes one or two arrays"))
    v = isempty(etc) ? nothing : etc[1]
    v === nothing || PencilArrays._check_compatible_arrays(u, v)
    map = pa_map(f)
    (map == 2 && v === nothing) || (map == 3 && v !== nothing) ||
        throw(ArgumentError("shell_spectrum: abs2 of one array or realdot of two, not $f"))
    H = handles(topology(pencil(u)))
    N = ndims(pencil(u))
    sc = scales === nothing ? C_NULL : Float64[s for s in scales]
    sc === C_NULL || length(sc) == N || throw(ArgumentError("shell_spectrum: one scale per dim"))
    nb = Ref{Cint}()
    GC.@preserve sc check(ccall((:pa_shell_spectrum_nbins, libpa), Cint,
        (Ptr{Cvoid}, Cint, Int64, Ptr{Float64}, Cdouble, Ptr{Cint}),
        pencil_handle(H, pencil(u)), rfft_dim, rfft_n, sc, width, nb))
    n = nbins === nothing ? Int(nb[]) : Int(nbins)
    result = CuVector{real(T)}(undef, max(n, 1))
    ex = Int64[extra_dims(u)...]
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    GC.@preserve sc check(ccall((:pa_shell_spectrum, libpa), Cint,
        (Ptr{Cvoid}, Cint, Ptr{Int64}, Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Int64,
         Ptr{Float64}, Cdouble, Cint, Ptr{Cvoid}, Ptr{Cvoid}),
        pencil_handle(H, pencil(u)), length(ex), ex, H.comm, PA_DTYPE[T], map,
        ptr_or_null(parent(u)), v === nothing ? C_NULL : ptr_or_null(parent(v)), rfft_dim, rfft_n,
        sc, width, n, devptr(result), stream_ptr()))
    result
end

function shell_spectrum_dims(f::F, u::CuPencilArray{T}, etc::Vararg{CuPencilArray{T}};
                             rfft_dim, rfft_n, scales, width, nbins, dims,
                             keep) where {F,T<:Union{ComplexF64,ComplexF32}}
    length(etc) <= 1 || throw(ArgumentError("shell_spectrum takes one or two arrays"))
    v = isempty(etc) ? nothing : etc[1]
    v === nothing || PencilArrays._check_compatible_arrays(u, v)
    map = pa_map(f)
    (map == 2 && v === nothing) || (map == 3 && v !== nothing) ||
        throw(ArgumentError("shell_spectrum: abs2 of one array or realdot of two, not $f"))
    H = handles(topology(pencil(u)))
    N = ndims(pencil(u))
    sc = scales === nothing ? C_NULL : Float64[s for s in scales]
    sc === C_NULL || length(sc) == N || throw(ArgumentError("shell_spectrum: one scale per dim"))
    bd = Cint[d for d in dims]
    kd = Cint[d for d in keep]
    nb = Ref{Cint}()
    GC.@preserve sc bd check(ccall((:pa_shell_spectrum_dims_nbins, libpa), Cint,
        (Ptr{Cvoid}, Cint, Int64, Ptr{Float64}, Cdouble, Cint, Ptr{Cint}, Ptr{Cint}),
        pencil_handle(H, pencil(u)), rfft_dim, rfft_n, sc, width, length(bd), bd, nb))
    n = nbins === nothing ? Int(nb[]) : Int(nbins)
    # the result: parent(u)'s local extents with every non-kept position 1, bins first (fastest)
    nl = ndims(parent(u))
    pp = permutation(pencil(u))
    perm = isidentity(pp) ? Tuple(1:N) : Tuple(pp)  # memory dim m holds logical dim perm[m]
    sz = ntuple(m -> (m <= N ? perm[m] : m) in keep ? size(parent(u), m) : 1, nl)
    result = CuArray{real(T)}(undef, max(n, 1), sz...)
    ex = Int64[extra_dims(u)...]
    ptr_or_null(A) = isempty(A) ? C_NULL : devptr(A)
    GC.@preserve sc bd kd check(ccall((:pa_shell_spectrum_dims, libpa), Cint,
        (Ptr{Cvoid}, Cint, Ptr{Int64}, Ptr{Cvoid}, Cint, Cint, Ptr{Cvoid}, Ptr{Cvoid}, Cint, Int64,
         Ptr{Float64}, Cdouble, Cint, Cint, Ptr{Cint}, Cint, Ptr{Cint}, Ptr{Cvoid}, Ptr{Cvoid}),
        pencil_handle(H, pencil(u)), length(ex), ex, H.comm, PA_DTYPE[T], map,
        ptr_or_null(parent(u)), v === nothing ? C_NULL : ptr_or_null(parent(v)), rfft_dim, rfft_n,
        sc, width, n, length(bd), bd, length(kd), kd, ptr_or_null(result), stream_ptr()))
    result
end

end # module
