"""``PencilIO``: the reference's MPI-IO driver surface (src/PencilIO/mpi_io.jl) over
libpa_b200 -- SURVEY.md §8(f4).

    with open_(MPIIODriver(), "fields.bin", comm, write=True, create=True) as ff:
        ff["velocity"] = (ux, uy, uz)            # setindex!(file, x, name)       :159-181
        ff.write("pressure", p, chunks=True)     # ... ; chunks, collective keywords
    with open_(MPIIODriver(), "fields.bin", comm, read=True) as ff:
        read_(ff, p, "pressure")                 # read!(file, x, name)           :236-259
        read_(ff, p)                             # metadata-less variant          :261-276

Files are byte-compatible with the reference's: raw binary (global array in the pencil's
memory order, or per-rank chunks) + a ``<filename>.json`` sidecar with the same keys
(:183-211).  Every rank moves its own part between device memory and the file
(``pa_io_write`` / ``pa_io_read``); rank 0 writes the sidecar on close.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import torch

from . import _lib
from ._lib import lib, check, i64arr, ArgumentError
from .arrays import PencilArray
from .pencils import MemoryOrder, LogicalOrder, size_global as _size_global
from .permutations import NoPermutation, as_tuple

MPIIO_VERSION = "0.9.4"  # mpi_io.jl:7
ENDIAN_BOM = "0x04030201"  # repr(ENDIAN_BOM) on a little-endian machine

_JULIA_TYPES = {torch.float32: "Float32", torch.float64: "Float64", torch.complex64: "ComplexF32",
                torch.complex128: "ComplexF64", torch.int8: "Int8", torch.int16: "Int16",
                torch.int32: "Int32", torch.int64: "Int64", torch.uint8: "UInt8", torch.float16: "Float16",
                torch.bool: "Bool"}


class MPIIODriver:  # mpi_io.jl:25-29
    def __init__(self, sequential=False, uniqueopen=False, deleteonclose=False):
        self.sequential, self.uniqueopen, self.deleteonclose = sequential, uniqueopen, deleteonclose


def _collection(x):
    return list(x) if isinstance(x, (tuple, list)) else [x]


def _collection_size(x):
    return (len(x),) if isinstance(x, (tuple, list)) else ()


def sizeof_global(x) -> int:
    """arrays.jl:423-429"""
    n = 0
    for u in _collection(x):
        g = 1
        for s in _size_global(u.pencil) + u.extra_dims:
            g *= s
        n += g * u.elsize
    return n


def _barrier(comm):
    import torch.distributed as dist
    if comm.size > 1 and dist.is_initialized():
        dist.barrier()


class MPIFile:
    """``MPIFile`` (mpi_io.jl:44-53): file name, metadata, position (bytes)."""

    def __init__(self, comm, filename, *, read=False, write=False, create=False, append=False,
                 truncate=False):
        if not (read or write):
            read = True
        self.comm, self.filename = comm, os.fspath(filename)
        self.write_mode = bool(write)
        self.position = 0
        metafile = self.filename + ".json"
        if write and not append:
            self.meta = {"driver": {"type": "MPIIODriver", "version": MPIIO_VERSION}, "datasets": {}}
            if comm.rank == 0:  # MPI.File.open(create=true) + position 0: start from an empty file
                with open(self.filename, "wb"):
                    pass
            _barrier(comm)
        else:
            if os.path.isfile(metafile):
                with open(metafile) as f:
                    m = json.load(f)
                self.meta = {"driver": m["driver"], "datasets": dict(m["datasets"])}
            elif write:
                self.meta = {"driver": {"type": "MPIIODriver", "version": MPIIO_VERSION}, "datasets": {}}
            else:
                self.meta = {}  # metadata file not found: assume a single dataset (:62-66)
            if append:
                self.position = os.path.getsize(self.filename) if os.path.exists(self.filename) else 0

    # ---- setindex!(file, x, name; chunks, collective) ----
    def write(self, name, x, *, chunks=False, collective=True):
        if not self.write_mode:
            raise ArgumentError(_lib.PA_EINVAL, "file was not opened for writing")
        offset = self.position
        for u in _collection(x):
            check(lib.pa_io_write(u.pencil._h, len(u.extra_dims), i64arr(u.extra_dims), u.elsize,
                                  1 if chunks else 0, C.c_void_p(u.data_ptr() or None),
                                  self.filename.encode(), offset))
            offset += sizeof_global(u)
        self._add_metadata(x, name, chunks)
        self.position += sizeof_global(x)
        return x

    def __setitem__(self, name, x):
        self.write(name, x)

    def _add_metadata(self, x, name, chunks):  # :183-211
        u = _collection(x)[0]
        pen = u.pencil
        perm = None if isinstance(pen.perm, NoPermutation) else list(as_tuple(pen.perm, pen.ndims))
        col = list(_collection_size(x))
        self.meta["datasets"][str(name)] = {
            "permutation": perm,
            "extra_dims": list(u.extra_dims),
            "decomposed_dims": list(pen.decomp_dims),
            "process_dims": list(pen.topology.dims),
            "julia_endian_bom": ENDIAN_BOM,
            "little_endian": True,
            "element_type": _JULIA_TYPES[u.dtype],
            "dims_logical": list(_size_global(pen, LogicalOrder())) + list(u.extra_dims) + col,
            "dims_memory": list(_size_global(pen, MemoryOrder())) + list(u.extra_dims) + col,
            "chunks": bool(chunks),
            "offset_bytes": int(self.position),
            "size_bytes": int(sizeof_global(x)),
        }

    def close(self):
        _barrier(self.comm)  # every rank's data is in the file before the metadata says so
        if self.write_mode and self.comm.rank == 0:
            with open(self.filename + ".json", "w") as f:
                json.dump(self.meta, f, indent=2)
                f.write("\n")
        _barrier(self.comm)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False


def open_(driver: MPIIODriver, filename, comm, **kw) -> MPIFile:
    """``open(MPIIODriver(), filename, comm; read, write, create, append)`` (:132-146)."""
    return MPIFile(comm, filename, **kw)


def read_(ff: MPIFile, x, name=None, *, offset=0, collective=True):
    """``read!(file, x, name)`` / ``read!(file, x; offset)`` (:236-290)."""
    chunks = False
    if name is not None:
        if not ff.meta:
            raise ArgumentError(_lib.PA_EINVAL, f"metadata file not found: {ff.filename}.json. Try calling "
                                "the `read_(ff, x)` variant (without the third argument) to attempt "
                                "reading the first dataset of the file.")
        meta = ff.meta["datasets"].get(str(name))
        if meta is None:
            raise RuntimeError(f"dataset '{name}' not found")
        _check_metadata(x, meta)
        offset, chunks = int(meta["offset_bytes"]), bool(meta["chunks"])
        if chunks:
            pd = tuple(_collection(x)[0].pencil.topology.dims)
            if tuple(meta["process_dims"]) != pd:
                raise RuntimeError(f"dataset '{name}' was written in chunks with a different MPI "
                                   f"topology ({pd} ≠ {tuple(meta['process_dims'])})")
    else:
        if sizeof_global(x) > os.path.getsize(ff.filename):
            raise RuntimeError("attempt to read file without JSON metadata failed: the file size is "
                               "inferior to the expected dataset size")
    for u in _collection(x):
        check(lib.pa_io_read(u.pencil._h, len(u.extra_dims), i64arr(u.extra_dims), u.elsize,
                             1 if chunks else 0, C.c_void_p(u.data_ptr() or None),
                             ff.filename.encode(), offset))
        offset += sizeof_global(u)
    return x


def _check_metadata(x, meta):  # :292-327
    u = _collection(x)[0]
    T = _JULIA_TYPES[u.dtype]
    if T != meta["element_type"]:
        raise RuntimeError(f"incompatible type of file and array: {meta['element_type']} ≠ {T}")
    sz = tuple(_size_global(u.pencil, MemoryOrder())) + u.extra_dims + _collection_size(x)
    if tuple(meta["dims_memory"]) != sz:
        raise RuntimeError("incompatible dimensions of dataset in file and array: "
                           f"{tuple(meta['dims_memory'])} ≠ {sz}")
    assert sizeof_global(x) == meta["size_bytes"]
    if int(str(meta.get("julia_endian_bom", ENDIAN_BOM)), 16) != int(ENDIAN_BOM, 16):
        raise RuntimeError("file was not written with the same native endianness of the current system. "
                           "Reading a non-native endianness is not yet supported.")
