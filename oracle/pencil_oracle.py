"""CPU ORACLE (test infrastructure -- never imported by the product path).

A NumPy restatement of the reference's `transpose!` path, written to follow
the Julia source function by function (file:line cited on each) with all MPI
ranks emulated inside one process.  Only `tests/`, `__graft_entry__.smoke()`
and the `cpu_baseline` / `--impl reference` legs of `bench.py` may import it.

Parity status: PINNED BY PROPERTIES, not by reference-produced outputs.
The reference is Julia + MPI and neither exists in this image, so it could not
be executed to produce golden outputs; its test-suite holds no golden vectors
either (every check is `gather(u) == gather(v)` or a round trip, see
test/transpose.jl:6-60).  This oracle is pinned against exactly those
properties plus the known-answer examples in the reference's docs/docstrings
(tests/test_oracle.py): docs/src/index.md:92-94, docs/src/Pencils.md:40-50,
src/arrays.jl:19-31.  Arithmetic is integer index math and byte moves only.

Conventions: 1-based inclusive index ranges as Python `range(a, b + 1)`;
arrays are NumPy arrays in Fortran (column-major) order, like Julia's.
"""
from __future__ import annotations

import itertools
import math

import numpy as np


# --------------------------------------------------------------------------- permutations
# StaticPermutations.jl v0.3 (third-party, not part of the reference); the
# semantics used are pinned by src/arrays.jl:19-31 and Transpositions.jl:503,524,599.
def perm_apply(p, t):
    """`p * t`: (p * t)[i] = t[p[i]]; p = None is NoPermutation."""
    if p is None:
        return tuple(t)
    return tuple(t[i - 1] for i in p)


def perm_rel(po, pi, n):
    """`po / pi`: position of po[i] in pi."""
    po = tuple(range(1, n + 1)) if po is None else po
    pi = tuple(range(1, n + 1)) if pi is None else pi
    return tuple(pi.index(v) + 1 for v in po)


def perm_inv(p):
    out = [0] * len(p)
    for i, v in enumerate(p):
        out[v - 1] = i + 1
    return tuple(out)


def perm_isidentity(p):
    return p is None or all(v == i + 1 for i, v in enumerate(p))


# --------------------------------------------------------------------------- data_ranges.jl
def local_data_range(p, P, N):
    """data_ranges.jl:4-9."""
    assert 1 <= p <= P
    a = (N * (p - 1)) // P + 1
    b = (N * p) // P
    return range(a, b + 1)


def complete_dims(N, dims, vals):
    """data_ranges.jl:15-26."""
    out = []
    for n in range(1, N + 1):
        out.append(vals[dims.index(n)] if n in dims else 1)
    return tuple(out)


def generate_axes_matrix(decomp_dims, proc_dims, size_global):
    """data_ranges.jl:30-45 -> dict: 1-based grid coords -> tuple of ranges."""
    N = len(size_global)
    procs = complete_dims(N, decomp_dims, proc_dims)
    axes = {}
    for I in itertools.product(*[range(1, d + 1) for d in proc_dims]):
        coords = complete_dims(N, decomp_dims, I)
        axes[I] = tuple(local_data_range(c, P, n) for c, P, n in zip(coords, procs, size_global))
    return axes


# --------------------------------------------------------------------------- MPITopologies.jl
def dims_create(nprocs, M):
    """MPI_Dims_create as used at MPITopologies.jl:138-144 (balanced, non-increasing)."""
    primes, n, f = [], nprocs, 2
    while f * f <= n:
        while n % f == 0:
            primes.append(f)
            n //= f
        f += 1
    if n > 1:
        primes.append(n)
    dims = [1] * M
    for pr in sorted(primes, reverse=True):
        dims[dims.index(min(dims))] *= pr
    return tuple(sorted(dims, reverse=True))


class OTopology:
    """MPITopology (MPITopologies.jl:72-119) of ONE rank; Cartesian ranks are
    row-major because the reference calls MPI.Cart_create(reorder=false) (:125-131)."""

    def __init__(self, dims, rank):
        self.dims = tuple(dims)
        self.rank = rank
        c, r = [], rank
        for d in reversed(self.dims):
            c.append(r % d + 1)
            r //= d
        self.coords_local = tuple(reversed(c))

    def rank_of(self, coords):
        r = 0
        for c, d in zip(coords, self.dims):
            r = r * d + (c - 1)
        return r


# --------------------------------------------------------------------------- Pencils.jl
class OPencil:
    """Pencil (Pencils.jl:151-272): geometry of one rank."""

    def __init__(self, topo: OTopology, size_global, decomp_dims, perm=None):
        self.topology = topo
        self.size_global = tuple(size_global)
        self.decomp_dims = tuple(decomp_dims)
        self.perm = None if perm_isidentity(perm) else tuple(perm)
        self.axes_all = generate_axes_matrix(self.decomp_dims, topo.dims, self.size_global)
        self.axes_local = self.axes_all[topo.coords_local]          # :228
        self.axes_local_perm = perm_apply(self.perm, self.axes_local)  # :229

    def size_local(self, memory_order=False):
        ax = self.axes_local_perm if memory_order else self.axes_local
        return tuple(len(r) for r in ax)

    def to_local(self, global_inds, memory_order=False):
        """Pencils.jl:579-587."""
        ind = tuple(range(rg.start + (1 - rl.start), rg.stop + (1 - rl.start))
                    for rg, rl in zip(global_inds, self.axes_local))
        return perm_apply(self.perm, ind) if memory_order else ind


class OArray:
    """PencilArray (arrays.jl:81-122): `data` in memory order, extra dims trailing."""

    def __init__(self, pencil: OPencil, data: np.ndarray, extra_dims=()):
        want = pencil.size_local(True) + tuple(extra_dims)
        if tuple(data.shape) != want:  # arrays.jl:108-114
            raise ValueError(f"DimensionMismatch: {data.shape} != {want}")
        self.pencil = pencil
        self.data = np.asfortranarray(data)
        self.extra_dims = tuple(extra_dims)

    @classmethod
    def undef(cls, dtype, pencil, *extra):
        return cls(pencil, np.zeros(pencil.size_local(True) + tuple(extra), dtype=dtype, order="F"),
                   extra)


def _isect(a, b):
    lo, hi = max(a.start, b.start), min(a.stop, b.stop)
    return range(lo, max(lo, hi))


def _sl(r):
    return slice(r.start - 1, r.stop - 1)


# --------------------------------------------------------------------------- Transpositions.jl
def assert_compatible(p: OPencil, q: OPencil):
    """Transpositions.jl:181-198 (topology identity is checked by the caller)."""
    if p.topology.dims != q.topology.dims:
        raise ValueError("ArgumentError: pencil topologies must be the same.")
    if p.size_global != q.size_global:
        raise ValueError("ArgumentError: global data sizes must be the same")
    if sum(a != b for a, b in zip(p.decomp_dims, q.decomp_dims)) > 1:
        raise ValueError("ArgumentError: pencil decompositions must differ in at most one dimension.")


def transposition_dim(Pi: OPencil, Po: OPencil):
    """Transpositions.jl:110: findfirst(decomposition(Pi) .!= decomposition(Po)); 1-based or None."""
    for i, (a, b) in enumerate(zip(Pi.decomp_dims, Po.decomp_dims)):
        if a != b:
            return i + 1
    return None


def get_remote_indices(R, coords_local, Nproc):
    """Transpositions.jl:539-549."""
    out = []
    for n in range(1, Nproc + 1):
        c = list(coords_local)
        c[R - 1] = n
        out.append(tuple(c))
    return out


def copy_range(dest, dest_offset, src: OArray, src_range_memorder):
    """copy_range! (Transpositions.jl:552-565): extra dims outermost, box column-major."""
    box = tuple(_sl(r) for r in src_range_memorder) + (slice(None),) * len(src.extra_dims)
    blk = src.data[box]
    n = blk.size
    dest[dest_offset:dest_offset + n] = blk.reshape(-1, order="F")
    return n


def copy_permuted(dst: OArray, o_range_iperm, src, src_offset, perm):
    """copy_permuted! -> _viewreshape -> _permutedims! (Transpositions.jl:585-645).
    `perm` = perm(Po) / perm(Pi) as a 1-based tuple over the spatial dims."""
    E = len(dst.extra_dims)
    src_dims = tuple(len(r) for r in o_range_iperm) + dst.extra_dims       # :596
    n = math.prod(src_dims)
    src_view = src[src_offset:src_offset + n].reshape(src_dims, order="F")  # :608-612
    dst_inds = perm_apply(perm, o_range_iperm)                              # :599
    box = tuple(_sl(r) for r in dst_inds) + (slice(None),) * E              # :627
    P = len(perm)
    pperm = tuple(perm) + tuple(range(P + 1, P + E + 1))                    # append(perm, Val(E)) :639
    # v .= permutedims(src, pperm): v[k] = src[j] with k[i] = j[pperm[i]]   (:633-645)
    dst.data[box] = np.transpose(src_view, tuple(i - 1 for i in pperm))
    return n


class RankState:
    """Buffers and bookkeeping of one emulated rank during one transpose!."""

    def __init__(self):
        self.send_buf = None
        self.recv_buf = None
        self.recv_offsets = None
        self.messages = []   # (peer_rank, send_off, send_len, recv_off, recv_len) in elements
        self.remote_inds = None
        self.index_local = None


def transpose_send(Ao: OArray, Ai: OArray, R: int, st: RankState):
    """transpose_impl!(R) sizes (:293-317) + transpose_send! (:345-430)."""
    Pi, Po = Ai.pencil, Ao.pencil
    topo = Pi.topology
    Nproc = topo.dims[R - 1]
    remote_inds = get_remote_indices(R, topo.coords_local, Nproc)
    prod_extra = math.prod(Ai.extra_dims)
    length_self = math.prod(len(_isect(a, b)) for a, b in zip(Pi.axes_local, Po.axes_local)) * prod_extra
    length_send = Ai.data.size - length_self            # :308
    length_recv_total = Ao.data.size                    # :309
    st.send_buf = np.zeros(max(1, length_send), dtype=Ai.data.dtype)
    st.recv_buf = np.zeros(max(1, length_recv_total), dtype=Ai.data.dtype)
    st.recv_offsets = [0] * Nproc
    st.remote_inds = remote_inds
    length_recv = Ao.data.size - length_self            # :372
    isend = irecv = 0
    myrank = topo.rank
    for n, ind in enumerate(remote_inds):
        srange = tuple(_isect(a, b) for a, b in zip(Pi.axes_local, Po.axes_all[ind]))   # :382
        length_send_n = math.prod(len(r) for r in srange) * prod_extra
        local_send_range = Pi.to_local(srange, memory_order=True)                        # :384
        rrange = tuple(_isect(a, b) for a, b in zip(Po.axes_local, Pi.axes_all[ind]))   # :387
        length_recv_n = math.prod(len(r) for r in rrange) * prod_extra
        st.recv_offsets[n] = irecv
        rank = topo.rank_of(ind)
        if rank == myrank:
            assert length_recv_n == length_self
            st.recv_offsets[n] = length_recv                                             # :398
            copy_range(st.recv_buf, length_recv, Ai, local_send_range)
            st.index_local = n
        else:
            copy_range(st.send_buf, isend, Ai, local_send_range)                         # :406
            st.messages.append((rank, isend, length_send_n, irecv, length_recv_n))
            irecv += length_recv_n
            isend += length_send_n
    assert isend == length_send and irecv == length_recv


def transpose_recv(Ao: OArray, Ai: OArray, st: RankState):
    """transpose_recv! (:486-533); block order is irrelevant to the result."""
    Pi, Po = Ai.pencil, Ao.pencil
    N = len(Pi.size_global)
    perm = perm_rel(Po.perm, Pi.perm, N)                                                  # :503
    order = [st.index_local] + [n for n in range(len(st.remote_inds)) if n != st.index_local]
    for n in order:
        ind = st.remote_inds[n]
        g_range = tuple(_isect(a, b) for a, b in zip(Po.axes_local, Pi.axes_all[ind]))    # :518
        off = st.recv_offsets[n]
        o_range_iperm = perm_apply(Pi.perm, Po.to_local(g_range, memory_order=False))     # :524
        copy_permuted(Ao, o_range_iperm, st.recv_buf, off, perm)


def permute_local(Ao: OArray, Ai: OArray):
    """transpose_impl!(::Nothing) + permute_local! (:213-270)."""
    Pi, Po = Ai.pencil, Ao.pencil
    N = len(Pi.size_global)
    if (Pi.perm or None) == (Po.perm or None):
        Ao.data[...] = Ai.data
        return
    E = len(Ai.extra_dims)
    perm = perm_rel(Po.perm, Pi.perm, N) + tuple(range(N + 1, N + E + 1))
    Ao.data[...] = np.transpose(Ai.data.copy(), tuple(i - 1 for i in perm))


def transpose_all(dests, srcs, keep_states=False):
    """`transpose!(dest, src)` executed by every rank of the grid; `dests` /
    `srcs` are lists indexed by world rank.  The exchange (Isend/Irecv or
    Alltoallv, :418-427,462-476) is a copy between the emulated ranks' buffers."""
    nranks = len(srcs)
    Pi0, Po0 = srcs[0].pencil, dests[0].pencil
    if srcs[0].extra_dims != dests[0].extra_dims:
        raise ValueError("ArgumentError: incompatible number of extra dimensions")
    assert_compatible(Pi0, Po0)
    R = transposition_dim(Pi0, Po0)
    if R is None:
        for r in range(nranks):
            permute_local(dests[r], srcs[r])
        return None
    states = [RankState() for _ in range(nranks)]
    for r in range(nranks):
        transpose_send(dests[r], srcs[r], R, states[r])
    for r in range(nranks):                       # deliver messages
        for (peer, soff, slen, _, _) in states[r].messages:
            # the matching receive on `peer` is the one posted for source rank r
            for (src_rank, _, _, roff, rlen) in states[peer].messages:
                if src_rank == r:
                    assert rlen == slen
                    states[peer].recv_buf[roff:roff + rlen] = states[r].send_buf[soff:soff + slen]
    for r in range(nranks):
        transpose_recv(dests[r], srcs[r], states[r])
    return states if keep_states else None


def gather(arrays):
    """gather (gather.jl:17-100): global array in logical order (+ extra dims)."""
    p0 = arrays[0].pencil
    extra = arrays[0].extra_dims
    N = len(p0.size_global)
    out = np.zeros(p0.size_global + extra, dtype=arrays[0].data.dtype, order="F")
    for a in arrays:
        pen = a.pencil
        data = a.data
        if pen.perm is not None:  # apply the inverse permutation (:32-40)
            ip = perm_inv(pen.perm) + tuple(range(N + 1, N + len(extra) + 1))
            data = np.transpose(data, tuple(i - 1 for i in ip))
        box = tuple(_sl(r) for r in pen.axes_local) + (slice(None),) * len(extra)
        out[box] = data
    return out


# --------------------------------------------------------------------------- helpers for tests / bench
def make_pencils(pdims, size_global, decomp_dims, perm=None):
    """One OPencil per world rank of a `pdims` process grid."""
    nranks = math.prod(pdims)
    return [OPencil(OTopology(pdims, r), size_global, decomp_dims, perm) for r in range(nranks)]


def splitmix64(x):
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    z = x
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def global_pattern(size_global, extra, itemsize, seed=42):
    """Synthetic global array (SURVEY.md §8d): element with 0-based column-major
    linear index `lin` holds splitmix64(word_index ^ seed) per 8-byte word
    (truncated for smaller elements).  Returned as raw bytes, shape
    size_global + extra + (itemsize,), Fortran order over the leading dims."""
    n = math.prod(size_global) * math.prod(extra)
    words = max(1, itemsize // 8)
    with np.errstate(over="ignore"):
        idx = np.arange(n * words, dtype=np.uint64) ^ np.uint64(seed)
        vals = splitmix64(idx)
    raw = vals.view(np.uint8).reshape(n * words, 8)
    if itemsize < 8:
        raw = raw[:, :itemsize]
    raw = raw.reshape(n, itemsize)
    return raw.reshape(tuple(size_global) + tuple(extra) + (itemsize,), order="F")


def scatter(global_bytes, pencils, extra, dtype):
    """Cut the global pattern into per-rank OArrays (memory order of each pencil)."""
    N = len(pencils[0].size_global)
    out = []
    for pen in pencils:
        box = tuple(_sl(r) for r in pen.axes_local) + (slice(None),) * (len(extra) + 1)
        loc = global_bytes[box]
        if pen.perm is not None:
            axes = tuple(i - 1 for i in pen.perm) + tuple(range(N, N + len(extra) + 1))
            loc = np.transpose(loc, axes)
        loc = np.ascontiguousarray(loc.reshape(-1, loc.shape[-1], order="F")).view(dtype).reshape(-1)
        data = loc.reshape(pen.size_local(True) + tuple(extra), order="F")
        out.append(OArray(pen, data, extra))
    return out
