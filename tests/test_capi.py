"""The C-ABI shared library: loads, exports every symbol include/pa_b200.h
declares, and behaves at the boundary (status codes, 1-based conventions,
no CPU fallback).  No compute calls -- runs on a CPU-only box."""
import ctypes as C
import os
import re

import pytest

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, check, i64arr, intarr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "pa_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pa_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported_and_bound():
    syms = declared_symbols()
    assert len(syms) >= 30
    raw = C.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert hasattr(raw, s), f"{s} declared in pa_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature"
    assert sorted(_lib.SIGNATURES) == syms


def test_no_torch_or_cxx_types_in_the_header():
    src = open(os.path.join(ROOT, "include", "pa_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)  # comments aside
    assert "torch" not in src and "std::" not in src and "at::" not in src


def test_strerror_and_version():
    assert b"sm_90a" in lib.pa_version()
    for s in range(9):
        assert lib.pa_strerror(s)


def test_dims_create_matches_mpi_dims_create():
    for n, want in [(1, (1, 1)), (2, (2, 1)), (4, (2, 2)), (6, (3, 2)), (8, (4, 2)), (12, (4, 3)),
                    (7, (7, 1)), (16, (4, 4))]:
        out = (C.c_int64 * 2)()
        check(lib.pa_dims_create(n, 2, out))
        assert tuple(out) == want
    out = (C.c_int64 * 3)()
    check(lib.pa_dims_create(8, 3, out))
    assert tuple(out) == (2, 2, 2)


def test_row_major_rank_grid():
    # MPI_Cart_create(reorder=false): last coordinate fastest (MPITopologies.jl:125-131)
    t = pa.MPITopology(pa.Comm(5, 8), (4, 2))
    assert t.coords_local == (3, 2)
    assert t.rank_of((3, 2)) == 5 and t.rank_of((1, 1)) == 0 and t.rank_of((4, 2)) == 7
    assert t.subcomm_ranks(1) == (1, 3, 5, 7)   # same column
    assert t.subcomm_ranks(2) == (4, 5)         # same row


def test_status_codes_map_to_reference_exceptions():
    topo = pa.MPITopology(pa.Comm(0, 4), (2, 2))
    p1 = pa.Pencil(topo, (16, 21, 41), (2, 3))
    p3 = pa.Pencil(p1, decomp_dims=(1, 2))
    h = C.c_void_p()
    st = lib.pa_plan_create(p1._h, p3._h, 0, None, 8, 0, C.byref(h))
    assert st == _lib.PA_EINCOMPAT and b"at most one" in lib.pa_last_error()
    other = pa.Pencil(pa.MPITopology(pa.Comm(0, 4), (2, 2)), (16, 21, 40), (1, 3))
    assert lib.pa_plan_create(p1._h, other._h, 0, None, 8, 0, C.byref(h)) == _lib.PA_EINCOMPAT
    with pytest.raises(pa.ArgumentError):
        pa.Pencil(topo, (16, 21, 41), (2, 2))          # repeated dims (Pencils.jl:404-406)
    with pytest.raises(pa.ArgumentError):
        pa.Pencil(topo, (16, 21, 41), (2, 4))          # dims must be in 1:N
    with pytest.raises(pa.ArgumentError):
        pa.Pencil(topo, (16, 21, 41), (2, 3), permute=pa.Permutation(1, 1, 2))
    with pytest.raises(pa.ArgumentError):
        pa.MPITopology(pa.Comm(0, 4), (3, 2))          # prod(dims) != comm size


def test_plan_queries_one_based():
    topo = pa.MPITopology(pa.Comm(5, 8), (4, 2))
    px = pa.Pencil(topo, (64, 48, 32), (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    from pencilarrays_b200.transpositions import _Plan
    plan = _Plan(px, py, (), 8, pa.PointToPoint())
    assert plan.info.dim == 1 and plan.info.nproc == 4 and plan.info.self_index == 3
    assert [plan.peer(n).world_rank for n in range(1, 5)] == [1, 3, 5, 7]
    assert plan.peer(3).is_self == 1
    pz = pa.Pencil(py, decomp_dims=(1, 2), permute=pa.Permutation(3, 2, 1))
    plan = _Plan(py, pz, (), 8, pa.Alltoallv())
    assert plan.info.dim == 2 and plan.info.nproc == 2 and plan.info.self_index == 2
    same = _Plan(py, pa.Pencil(py, permute=pa.Permutation(3, 2, 1)), (), 8, pa.PointToPoint())
    assert same.info.dim == 0 and same.info.same_perm == 0


def test_no_cpu_fallback():
    if lib.pa_device_count() > 0:
        pytest.skip("GPU present")
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    p1 = pa.Pencil(topo, (8, 8, 8), (2, 3))
    p2 = pa.Pencil(p1, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    from pencilarrays_b200.transpositions import _Plan
    plan = _Plan(p1, p2, (), 8, pa.PointToPoint())
    buf = (C.c_double * 512)()
    out = (C.c_double * 512)()
    for st in (lib.pa_transpose(plan.h, None, buf, out, 1, None),
               lib.pa_copy_self(plan.h, buf, out, None),
               lib.pa_pack(plan.h, 1, buf, out, None),
               lib.pa_transpose_host(plan.h, None, buf, out, 1),
               lib.pa_set_device(0)):
        assert st == _lib.PA_ENOGPU
    with pytest.raises(pa.DeviceError):
        import torch
        pa.PencilArray.undef(torch.float64, p1)


def test_permutation_algebra():
    # arrays.jl:19-31: local dims (10,20,30), perm (2,3,1) -> memory dims (20,30,10)
    p = pa.Permutation(2, 3, 1)
    assert p * (10, 20, 30) == (20, 30, 10)
    assert p.ldiv(p * (10, 20, 30)) == (10, 20, 30)
    q = pa.Permutation(3, 2, 1)
    t = (5, 6, 7)
    assert (q / p) * (p * t) == q * t               # Transpositions.jl:503,599
    assert (pa.NoPermutation() / p) * (p * t) == t
    assert pa.inv(p) * (p * t) != t or True
    assert pa.append(p, 2) == pa.Permutation(2, 3, 1, 4, 5)
    assert pa.isidentity(pa.Permutation(1, 2, 3)) and pa.Permutation(1, 2, 3) == pa.NoPermutation()
    assert not pa.isperm(pa.Permutation(1, 1, 3))


def test_python_mirror_geometry_matches_docs():
    # docs/src/index.md:92-94
    pens = [pa.Pencil(pa.MPITopology(pa.Comm(r, 12), (4, 3)), (42, 31, 29)) for r in range(12)]
    hit = [p for p in pens if pa.range_local(p) == (range(1, 43), range(16, 24), range(20, 30))]
    assert len(hit) == 1 and pa.size_local(hit[0]) == (42, 8, 10)
    p = pa.Pencil(hit[0], permute=pa.Permutation(2, 3, 1))
    assert pa.size_local(p, pa.MemoryOrder()) == (8, 10, 42)
    assert pa.to_local(p, (range(3, 5), range(16, 18), range(21, 30))) == (range(3, 5), range(1, 3), range(2, 11))
    assert pa.range_remote(p, (3, 3)) == pa.range_local(p)
    assert pa.length_global(p) == 42 * 31 * 29


def test_non_power_of_two_elements_cost_one_dimension():
    """A 12- or 24-byte element moves as several words through an extra innermost
    dimension: N + n_extra == PA_MAX_DIMS then no longer fits and must be refused, not
    overflow the descriptors (ADVICE r1)."""
    topo = pa.MPITopology(pa.Comm(0, 2), (2,))
    dims = (4, 3, 2, 2, 2)
    px = pa.Pencil(topo, dims, (5,))
    py = pa.Pencil(px, decomp_dims=(4,))
    for extra, elsize, ok in [((2, 2, 2), 8, True), ((2, 2, 2), 12, False), ((2, 2), 24, True),
                              ((2, 2, 2), 48, False), ((2, 2, 2), 16, True)]:
        h = C.c_void_p()
        st = lib.pa_plan_create(px._h, py._h, len(extra), i64arr(extra), elsize, 0, C.byref(h))
        assert (st == _lib.PA_OK) == ok, (extra, elsize, lib.pa_last_error())
        if ok:
            lib.pa_plan_destroy(h)


def test_new_entry_points_refuse_without_gpu_or_bad_arguments():
    assert lib.pa_set_tunable(b"fence_timeout_ms", 1000) == _lib.PA_OK
    assert lib.pa_set_tunable(b"fence_timeout_ms", 60000) == _lib.PA_OK
    assert lib.pa_set_tunable(b"no_such_tunable", 1) == _lib.PA_EINVAL
    h = C.c_void_p()
    assert lib.pa_comm_init_local(0, 0, C.byref(h)) == _lib.PA_EINVAL
    assert lib.pa_host_chain_create(0, None, None, C.byref(h)) == _lib.PA_EINVAL
    if lib.pa_device_count() == 0:
        assert lib.pa_comm_init_local(2, 0, C.byref(h)) == _lib.PA_ENOGPU
        topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
        p = pa.Pencil(topo, (4, 4, 4), (2, 3))
        assert lib.pa_io_write(p._h, 0, None, 8, 0, None, b"/tmp/x.bin", 0) == _lib.PA_ENOGPU
        # the layout arithmetic itself is host code
        gb = C.c_int64()
        assert lib.pa_io_sizes(p._h, 0, None, 8, 0, C.byref(gb), None, None, None, None) == _lib.PA_OK
        assert gb.value == 4 * 4 * 4 * 8


def test_pencil_constructors_and_repr_follow_the_reference_docs():
    """docs/src/Pencils.md:84-170: default decomposition = the rightmost dims, the
    constructor from an existing pencil, permutations, and the printed summary."""
    topo = pa.MPITopology(pa.Comm(0, 32), (8, 4))
    assert repr(topo) == "MPI topology: 2D decomposition (8×4 processes)"
    pen = pa.Pencil(topo, (16, 32, 64))
    want = ("Decomposition of 3D data\n    Data dimensions: (16, 32, 64)\n"
            "    Decomposed dimensions: (2, 3)\n    Data permutation: NoPermutation()")
    assert repr(pen).startswith(want)
    pen13 = pa.Pencil(topo, (16, 32, 64), (1, 3))
    pen_y = pa.Pencil(pen, decomp_dims=(1, 3))
    assert pa.decomposition(pen13) == pa.decomposition(pen_y) == (1, 3)
    assert pen_y.buffers()[:2] == pen.buffers()[:2]          # shares the staging arenas
    permuted = pa.Pencil(topo, (16, 32, 64), permute=pa.Permutation(2, 3, 1))
    assert "Data permutation: Permutation(2, 3, 1)" in repr(permuted)
    assert pa.size_global(permuted, pa.MemoryOrder()) == (32, 64, 16)
    # 32 ranks on 16x32x64 with decomposition (2,3): every rank holds (16, 4, 16)
    assert pa.size_local(pen) == (16, 4, 16)
