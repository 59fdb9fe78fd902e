# test_b200_transpose.jl -- pins libpa_b200 against the REAL reference.
#
# NOT EXECUTED IN THIS REPOSITORY (no Julia / MPI in the build image).  For a
# maintainer with Julia, MPI, CUDA.jl and >= 1 H100:
#
#     mpiexec -n 8 julia --project test_b200_transpose.jl
#
# Every rank runs the reference's own CPU `transpose!` (Array storage, MPI
# transport) and the GPU path (CuArray storage, this library) on identical
# inputs and compares the parent arrays byte for byte -- the check this
# repository can only make against its CPU oracle (oracle/pencil_oracle.py).
using MPI
using PencilArrays
using PencilArrays.Transpositions: Transposition, PointToPoint, Alltoallv
using CUDA
using Random
using Test

include("B200PencilArrays.jl")
using .B200PencilArrays

MPI.Init()
comm = MPI.COMM_WORLD
rank = MPI.Comm_rank(comm)
CUDA.device!(rank % length(CUDA.devices()))

function same_bytes(a::Array, b::CuArray)
    reinterpret(UInt8, vec(a)) == reinterpret(UInt8, vec(Array(b)))
end

function run_case(dims, T; extra = ())
    # CPU pencils (reference) and device pencils (this library) with the same geometry
    pen1 = Pencil(dims, (2, 3), comm)
    pen2 = Pencil(pen1; decomp_dims = (1, 3), permute = Permutation(2, 3, 1))
    pen3 = Pencil(pen2; decomp_dims = (1, 2), permute = Permutation(3, 2, 1))
    gpen1 = Pencil(CuArray, dims, (2, 3), comm)
    gpen2 = Pencil(gpen1; decomp_dims = (1, 3), permute = Permutation(2, 3, 1))
    gpen3 = Pencil(gpen2; decomp_dims = (1, 2), permute = Permutation(3, 2, 1))

    u1 = PencilArray{T}(undef, pen1, extra...)
    randn!(MersenneTwister(42 + rank), u1)          # test/transpose.jl:38-41
    u1 .+= 10 * rank
    g1 = PencilArray{T}(undef, gpen1, extra...)
    copyto!(parent(g1), parent(u1))

    for method in (PointToPoint(), Alltoallv(), B200PencilArrays.PeerPut())
        u2 = PencilArray{T}(undef, pen2, extra...); u3 = PencilArray{T}(undef, pen3, extra...)
        g2 = PencilArray{T}(undef, gpen2, extra...); g3 = PencilArray{T}(undef, gpen3, extra...)
        cpu_method = method isa B200PencilArrays.PeerPut ? PointToPoint() : method
        transpose!(u2, u1; method = cpu_method)
        transpose!(u3, u2; method = cpu_method)
        t12 = Transposition(g2, g1; method)
        t23 = Transposition(g3, g2; method)
        if method isa B200PencilArrays.PeerPut
            B200PencilArrays.register_window!(t12)
            B200PencilArrays.register_window!(t23)
        end
        transpose!(t12)
        transpose!(t23; waitall = false)
        MPI.Waitall(t23)
        CUDA.synchronize()
        @test same_bytes(parent(u2), parent(g2))
        @test same_bytes(parent(u3), parent(g3))
    end
end

@testset "libpa_b200 == PencilArrays.jl CPU path (bit-exact)" begin
    run_case((16, 21, 41), Float64)                  # test/transpose.jl
    run_case((16, 21, 41), Float32; extra = (3, 4))  # test/pencils.jl:460-480
    run_case((64, 48, 32), ComplexF64)
end

MPI.Finalize()
