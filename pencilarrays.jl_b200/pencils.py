"""Host-side mirror of the reference's ``MPITopology`` and ``Pencil`` types
(src/Pencils/MPITopologies.jl, src/Pencils/Pencils.jl) -- same names, argument
meaning and error behaviour, for the part of their interface that
``transpose!`` and its callers use.  All geometry is computed by libpa_b200
(``pa_topology_*`` / ``pa_pencil_*``); this file holds no arithmetic of its own
beyond tuple shuffling.  Indices and ranges are 1-based inclusive (Python
``range(lo, hi + 1)`` objects), as in the reference.
"""
from __future__ import annotations

import ctypes as C
import math

from . import _lib
from ._lib import lib, check, i64arr, intarr, ArgumentError
from .comm import Comm
from .permutations import (AbstractPermutation, NoPermutation, Permutation, as_tuple, isperm,
                           isidentity)


class AbstractIndexOrder:
    pass


class MemoryOrder(AbstractIndexOrder):  # index_orders.jl:17
    pass


class LogicalOrder(AbstractIndexOrder):  # index_orders.jl:25
    pass


def _is_mem(order) -> bool:
    if isinstance(order, type):
        order = order()
    return isinstance(order, MemoryOrder)


class MPITopology:
    """``MPITopology(comm, dims)`` / ``MPITopology(comm, Val(M))``
    (MPITopologies.jl:72-144).  Ranks map to coordinates row-major, exactly as
    ``MPI.Cart_create(comm, dims; reorder=false)`` does."""

    def __init__(self, comm: Comm, dims):
        if isinstance(dims, int):  # Val(M): balanced grid (dims_create, :138-144)
            M = dims
            out = (C.c_int64 * M)()
            check(lib.pa_dims_create(comm.size, M, out))
            dims = tuple(out)
        dims = tuple(int(d) for d in dims)
        if math.prod(dims) != comm.size:  # check_topology (:146-153)
            raise ArgumentError(_lib.PA_EINVAL,
                                f"total number of processes ({comm.size}) must be equal to "
                                f"the product of `dims` {dims}")
        self.comm = comm
        self.dims = dims
        h = C.c_void_p()
        check(lib.pa_topology_create(len(dims), i64arr(dims), comm.rank, C.byref(h)))
        self._h = h
        coords = (C.c_int64 * len(dims))()
        check(lib.pa_topology_info(h, None, None, None, None, coords))
        self.coords_local = tuple(coords)

    def __del__(self):
        try:
            lib.pa_topology_destroy(self._h)
        except Exception:
            pass

    def __len__(self):
        return self.comm.size

    @property
    def ndims(self):
        return len(self.dims)

    def rank_of(self, coords) -> int:
        r = C.c_int()
        check(lib.pa_topology_rank_of(self._h, i64arr(coords), C.byref(r)))
        return r.value

    def subcomm_ranks(self, R: int):
        """World ranks of the grid line through the local coords along dim R (1-based)."""
        n = self.dims[R - 1]
        out = (C.c_int * n)()
        check(lib.pa_topology_line(self._h, R, out))
        return tuple(out)

    def __repr__(self):
        return f"MPI topology: {len(self.dims)}D decomposition ({'×'.join(map(str, self.dims))} processes)"


def get_comm(x):
    return x.comm if isinstance(x, MPITopology) else x.topology.comm


def coords_local(t: MPITopology):
    return t.coords_local


def default_decomposition(N: int, M: int):
    """Pencils.jl:389-392: the last M dimensions."""
    assert 0 < M <= N
    return tuple(N - M + d for d in range(1, M + 1))


class Pencil:
    """``Pencil(topology, size_global, decomp_dims; permute)`` and
    ``Pencil(p; decomp_dims, size_global, permute)`` (Pencils.jl:238-271); also
    ``Pencil(size_global, [decomp_dims], comm)`` (:274-280).

    Pencils derived from another pencil share its staging buffers
    (``send_buf`` / ``recv_buf``, device arenas owned by libpa_b200).
    """

    def __init__(self, *args, decomp_dims=None, size_global=None, permute=None):
        parent = None
        if len(args) >= 1 and isinstance(args[0], Pencil):
            parent = args[0]
            topology = parent.topology
            size_global = parent.size_global if size_global is None else tuple(size_global)
            decomp_dims = parent.decomp_dims if decomp_dims is None else tuple(decomp_dims)
            permute = parent.perm if permute is None else permute
        elif len(args) >= 2 and isinstance(args[0], MPITopology):
            topology = args[0]
            size_global = tuple(args[1])
            if len(args) >= 3:
                decomp_dims = tuple(args[2])
        elif len(args) >= 2 and isinstance(args[-1], Comm):
            size_global = tuple(args[0])
            comm = args[-1]
            if len(args) == 3:
                decomp_dims = tuple(args[1])
                M = len(decomp_dims)
            else:
                M = len(size_global) - 1
                decomp_dims = default_decomposition(len(size_global), M)
            topology = MPITopology(comm, M)
        else:
            raise TypeError("Pencil(topology, size_global[, decomp_dims]) | Pencil(pencil; ...) | "
                            "Pencil(size_global[, decomp_dims], comm)")
        N = len(size_global)
        M = topology.ndims
        if decomp_dims is None:
            decomp_dims = default_decomposition(N, M)
        decomp_dims = tuple(int(d) for d in decomp_dims)
        if len(decomp_dims) != M:
            raise ArgumentError(_lib.PA_EINVAL,
                                f"decomp_dims {decomp_dims} must have {M} entries")
        permute = NoPermutation() if permute is None else permute
        if not isinstance(permute, AbstractPermutation) or not isperm(permute) or (
                isinstance(permute, Permutation) and len(permute) != N):
            raise ArgumentError(_lib.PA_EINVAL, f"invalid permutation of dimensions: {permute}")
        self.topology = topology
        self.size_global = tuple(int(s) for s in size_global)
        self.decomp_dims = decomp_dims
        self.perm = permute
        h = C.c_void_p()
        perm_arr = None if isinstance(permute, NoPermutation) else intarr(as_tuple(permute, N))
        check(lib.pa_pencil_create(topology._h, N, i64arr(self.size_global), intarr(decomp_dims),
                                   perm_arr, parent._h if parent is not None else None,
                                   C.byref(h)))
        self._h = h
        self._family = parent._family if parent is not None else self  # owner of the buffers
        self._plans = {}
        self.axes_local = self._range(None, False)
        self.axes_local_perm = self._range(None, True)

    def __del__(self):
        try:
            self._plans.clear()
            lib.pa_pencil_destroy(self._h)
        except Exception:
            pass

    # ---- geometry (all from the C library) ----
    def _range(self, coords, memory_order: bool):
        N = len(self.size_global)
        lo = (C.c_int64 * N)()
        hi = (C.c_int64 * N)()
        check(lib.pa_pencil_range(self._h, None if coords is None else i64arr(coords),
                                  1 if memory_order else 0, lo, hi))
        return tuple(range(l, h + 1) for l, h in zip(lo, hi))

    @property
    def ndims(self):
        return len(self.size_global)

    def buffers(self):
        """(send_ptr, send_capacity, recv_ptr, recv_capacity) of the shared device arenas."""
        sp, rp = C.c_void_p(), C.c_void_p()
        sc, rc = C.c_int64(), C.c_int64()
        check(lib.pa_pencil_buffers(self._h, C.byref(sp), C.byref(sc), C.byref(rp), C.byref(rc)))
        return sp.value, sc.value, rp.value, rc.value

    def __repr__(self):
        return ("Decomposition of {}D data\n    Data dimensions: {}\n    Decomposed dimensions: {}\n"
                "    Data permutation: {}\n    Array type: CUDA device memory (H100)").format(
                    self.ndims, self.size_global, self.decomp_dims, self.perm)


# ---- accessor functions, named as in Pencils.jl ----
def topology(p: Pencil):
    return p.topology


def decomposition(p: Pencil):
    return p.decomp_dims


def permutation(p):
    return p.perm if isinstance(p, Pencil) else p.pencil.perm


def range_local(p: Pencil, order=LogicalOrder()):
    return p.axes_local_perm if _is_mem(order) else p.axes_local


def range_remote(p: Pencil, coords, order=LogicalOrder()):
    if isinstance(coords, int):  # linear index into the (column-major) process grid, 1-based
        n = coords - 1
        c = []
        for d in p.topology.dims:
            c.append(n % d + 1)
            n //= d
        coords = tuple(c)
    return p._range(tuple(coords), _is_mem(order))


def size_local(p: Pencil, order=LogicalOrder()):
    return tuple(len(r) for r in range_local(p, order))


def size_global(p: Pencil, order=LogicalOrder()):
    return p.perm * p.size_global if _is_mem(order) else p.size_global


def length_local(p: Pencil):
    return math.prod(size_local(p))


def length_global(p: Pencil):
    return math.prod(p.size_global)


def to_local(p: Pencil, global_inds, order=LogicalOrder()):
    """Pencils.jl:579-587: logical global ranges -> local ranges."""
    ind = tuple(range(rg.start + 1 - rl.start, rg.stop + 1 - rl.start)
                for rg, rl in zip(global_inds, p.axes_local))
    return p.perm * ind if _is_mem(order) else ind
