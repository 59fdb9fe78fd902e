"""`pa_r2r` at the C-ABI boundary on HOST buffers: the symbol is exported and bound, every refusal
is decided on the host before any device call, and valid arguments without a device give
PA_ENOGPU.  Plus the argument checks of the Python `r2r_`.  No compute calls -- runs on a CPU-only
box."""
import ctypes as C

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, i64arr

KINDS = (_lib.PA_REDFT10, _lib.PA_REDFT01, _lib.PA_RODFT10, _lib.PA_RODFT01)
F32 = _lib.PA_FFT_F32


class HostBuf:
    """16-byte-aligned host memory (the checks only look at addresses and sizes)."""

    def __init__(self, nbytes):
        self.raw = np.zeros(nbytes + 64, dtype=np.uint8)
        a = self.raw.ctypes.data
        self.addr = a + (-a) % 16

    def at(self, off=0):
        return C.c_void_p(self.addr + off)


def pencil(dims=(16, 6, 4), decomp=(2, 3), perm=None, topo=None):
    topo = topo or pa.MPITopology(pa.COMM_SELF, (1, 1))
    return pa.Pencil(topo, dims, decomp, permute=pa.Permutation(*perm) if perm else None)


def nbytes(p, extra=(), flags=0):
    return int(np.prod(pa.size_local(p))) * int(np.prod(extra)) * (4 if flags & F32 else 8)


def call(p, kind=_lib.PA_REDFT10, flags=0, extra=(), src=None, dst=None, n_extra=None, extra_ptr=True):
    if src is None or dst is None:
        n = nbytes(p, extra, flags)
        a, b = HostBuf(n), HostBuf(n)
        call.keep = (a, b)
        src, dst = a.at(), b.at()
    n_extra = len(extra) if n_extra is None else n_extra
    return lib.pa_r2r(p._h, n_extra, i64arr(extra) if extra_ptr else None, kind, flags, src, dst, None)


def no_gpu():
    return lib.pa_device_count() == 0


def test_exported_and_bound():
    assert "pa_r2r" in _lib.SIGNATURES
    assert lib.pa_r2r.argtypes == _lib.SIGNATURES["pa_r2r"][1]
    # FFTW's fftw_r2r_kind values
    assert (_lib.PA_REDFT01, _lib.PA_REDFT10, _lib.PA_RODFT01, _lib.PA_RODFT10) == (4, 5, 8, 9)
    assert pa.r2r_ is pa.Transpositions.r2r_


@pytest.mark.parametrize("flags", [0, F32])
@pytest.mark.parametrize("kw", [dict(), dict(perm=(1, 3, 2)), dict(dims=(2048, 3, 2)),
                                dict(dims=(6, 32, 4), perm=(2, 1, 3), decomp=(1, 3)),
                                dict(dims=(16, 0, 4))])
def test_valid_arguments_without_a_device_give_enogpu(flags, kw):
    if not no_gpu():
        pytest.skip("GPU present")
    p = pencil(**kw)
    for kind in KINDS:
        assert call(p, kind, flags) == _lib.PA_ENOGPU
        assert call(p, kind, flags, extra=(2,)) == _lib.PA_ENOGPU


def test_in_place_and_null_pointers_of_an_empty_array_are_accepted():
    if not no_gpu():
        pytest.skip("GPU present")
    p = pencil()
    buf = HostBuf(nbytes(p))
    assert lib.pa_r2r(p._h, 0, None, _lib.PA_REDFT10, 0, buf.at(), buf.at(), None) == _lib.PA_ENOGPU
    e = pencil(dims=(16, 0, 4))
    assert lib.pa_r2r(e._h, 0, None, _lib.PA_REDFT01, 0, None, None, None) == _lib.PA_ENOGPU


def test_null_pencil():
    assert lib.pa_r2r(None, 0, None, _lib.PA_REDFT10, 0, None, None, None) == _lib.PA_EINVAL
    assert b"null pencil" in lib.pa_last_error()


@pytest.mark.parametrize("kw", [dict(decomp=(1, 3)), dict(perm=(2, 1, 3), decomp=(2, 3)),
                                dict(perm=(3, 1, 2), decomp=(1, 3))])
def test_decomposed_transform_axis(kw):
    p = pencil(**kw)
    for kind in KINDS:
        assert call(p, kind) == _lib.PA_EINCOMPAT, kw
        assert b"decomposed" in lib.pa_last_error()


def test_bad_kind_or_flags():
    p = pencil()
    for kind in (0, 1, 2, 3, 6, 7, 10, -1, 5 | 32):
        assert call(p, kind) == _lib.PA_EINVAL, kind
        assert b"kind" in lib.pa_last_error()
    for flags in (_lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD, _lib.PA_WAITALL, F32 | 1, 64):
        assert call(p, _lib.PA_REDFT10, flags) == _lib.PA_EINVAL, flags
        assert b"flags" in lib.pa_last_error()


@pytest.mark.parametrize("n", [8, 24, 4096, 2])
def test_line_length_not_a_power_of_two_in_16_to_2048(n):
    p = pencil(dims=(n, 4, 4))
    for flags in (0, F32):
        assert call(p, _lib.PA_RODFT10, flags) == _lib.PA_EINVAL
        assert b"power of two" in lib.pa_last_error()


def test_null_pointers_for_non_empty_arrays():
    p = pencil()
    buf = HostBuf(nbytes(p))
    for src, dst in ((None, buf.at()), (buf.at(), None), (None, None)):
        assert lib.pa_r2r(p._h, 0, None, _lib.PA_REDFT10, 0, src, dst, None) == _lib.PA_EINVAL
        assert b"null" in lib.pa_last_error()


@pytest.mark.parametrize("flags", [0, F32])
def test_partial_overlap_and_alignment(flags):
    p = pencil()
    n = nbytes(p, (), flags)
    buf = HostBuf(2 * n + 64)
    # overlapping by one 16-byte step either way (in place, src == dst, is allowed)
    for s, d in ((0, n - 16), (n - 16, 0), (0, 16), (16, 0)):
        assert call(p, _lib.PA_REDFT10, flags, src=buf.at(s), dst=buf.at(d)) == _lib.PA_EINVAL, (s, d)
        assert b"overlap" in lib.pa_last_error()
    # misaligned by 8 (4) bytes, apart or in place
    for s, d in ((8, n + 16), (0, n + 8), (4, n + 16), (8, 8)):
        assert call(p, _lib.PA_REDFT01, flags, src=buf.at(s), dst=buf.at(d)) == _lib.PA_EINVAL, (s, d)
        assert b"aligned" in lib.pa_last_error()
    if no_gpu():
        assert call(p, _lib.PA_REDFT10, flags, src=buf.at(0), dst=buf.at(n)) == _lib.PA_ENOGPU
        assert call(p, _lib.PA_REDFT10, flags, src=buf.at(16), dst=buf.at(16)) == _lib.PA_ENOGPU


def test_extra_dims_limits():
    p = pencil()
    if no_gpu():
        assert call(p, extra=(1, 1, 1, 1, 2)) == _lib.PA_ENOGPU    # 3 + 5 = PA_MAX_DIMS
    assert call(p, extra=(1, 1, 1, 1, 1, 2)) == _lib.PA_EINVAL     # 3 + 6 > PA_MAX_DIMS
    assert b"extra dims" in lib.pa_last_error()
    assert call(p, extra=(2,), extra_ptr=False) == _lib.PA_EINVAL  # NULL extra_dims
    assert call(p, extra=(2,), n_extra=-1) == _lib.PA_EINVAL
    buf = HostBuf(1 << 14)
    assert call(p, extra=(-2,), src=buf.at(0), dst=buf.at(1 << 13)) == _lib.PA_EINVAL
    assert b"negative" in lib.pa_last_error()


def test_order_of_the_checks_follows_pa_rfft():
    """Decomposed axis before a bad kind, a bad kind before a bad N, a bad N before the extra dims,
    the extra dims before the pointers."""
    assert call(pencil(decomp=(1, 3)), kind=0) == _lib.PA_EINCOMPAT
    assert b"decomposed" in lib.pa_last_error()
    assert call(pencil(dims=(24, 4, 4)), kind=0) == _lib.PA_EINVAL
    assert b"kind" in lib.pa_last_error()
    assert call(pencil(dims=(24, 4, 4)), extra=(1,) * 6) == _lib.PA_EINVAL
    assert b"power of two" in lib.pa_last_error()
    p = pencil()
    assert lib.pa_r2r(p._h, 6, i64arr((1,) * 6), _lib.PA_REDFT10, 0, None, None, None) == _lib.PA_EINVAL
    assert b"extra dims" in lib.pa_last_error()


def test_python_wrapper_checks_dtypes_geometry_and_extra_dims():
    """The checks of r2r_ run before anything touches a device (CPU tensors stand in for the
    parent arrays here)."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    p = pencil(topo=topo)

    def arr(q, dtype, *extra):
        mem = pa.size_local(q, pa.MemoryOrder())
        return pa.PencilArray(q, torch.zeros(tuple(reversed(mem + extra)), dtype=dtype), extra)

    x = arr(p, torch.float64)
    # the same geometry on another Pencil object is the same geometry
    assert pa.Transpositions._same_geometry(pencil(topo=topo), p)
    for a, b in ((arr(p, torch.float32), x), (x, arr(p, torch.float32)),
                 (arr(p, torch.complex128), arr(p, torch.complex128)),
                 (arr(p, torch.complex64), arr(p, torch.complex64)),
                 (arr(p, torch.int64), arr(p, torch.int64))):
        with pytest.raises(pa.ArgumentError):
            pa.r2r_(a, b, "REDFT10")
    with pytest.raises(pa.ArgumentError):
        pa.r2r_(x, x, "REDFT00")
    with pytest.raises(pa.ArgumentError):
        pa.r2r_(x, x, 5)
    # mismatched pencils: another size, permutation, decomposition or topology object
    for q in (pencil(dims=(32, 6, 4), topo=topo), pencil(perm=(1, 3, 2), topo=topo),
              pencil(decomp=(3, 2), topo=topo), pencil()):
        with pytest.raises(pa.ArgumentError):
            pa.r2r_(arr(q, torch.float64), x, "REDFT01")
    with pytest.raises(pa.ArgumentError):
        pa.r2r_(arr(p, torch.float64, 2), arr(p, torch.float64, 3), "RODFT10")
    with pytest.raises(pa.ArgumentError):
        pa.r2r_(arr(p, torch.float32), arr(p, torch.float32, 2), "RODFT01")
