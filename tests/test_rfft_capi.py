"""`pa_rfft` at the C-ABI boundary on HOST buffers: every refusal is decided on the host before
any device call, valid arguments without a device give PA_ENOGPU.  Plus the argument checks of
the Python `rfft_` / `brfft_`.  No compute calls -- runs on a CPU-only box."""
import ctypes as C

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, i64arr

FWD, BWD = _lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD


class HostBuf:
    """16-byte-aligned host memory (the checks only look at addresses and sizes)."""

    def __init__(self, nbytes):
        self.raw = np.zeros(nbytes + 64, dtype=np.uint8)
        a = self.raw.ctypes.data
        self.addr = a + (-a) % 16

    def at(self, off=0):
        return C.c_void_p(self.addr + off)


def pencils(real_dims=(16, 6, 4), cplx_dims=None, decomp=(2, 3), perm=None, cdecomp=None, cperm=None,
            topo=None, ctopo=None):
    topo = topo or pa.MPITopology(pa.COMM_SELF, (1, 1))
    permute = pa.Permutation(*perm) if perm else None
    pr = pa.Pencil(topo, real_dims, decomp, permute=permute)
    if cplx_dims is None:
        ax = (perm or (1, 2, 3))[0] - 1
        cplx_dims = tuple(n // 2 + 1 if d == ax else n for d, n in enumerate(real_dims))
    cpermute = pa.Permutation(*cperm) if cperm else permute
    if ctopo is not None:
        pc = pa.Pencil(ctopo, cplx_dims, cdecomp or decomp, permute=cpermute)
    else:
        pc = pa.Pencil(pr, size_global=cplx_dims, decomp_dims=cdecomp or decomp, permute=cpermute)
    return pr, pc


def call(pr, pc, flags=FWD, extra=(), src=None, dst=None, n_extra=None, extra_ptr=True):
    ncols = 1
    for n in extra:
        ncols *= n
    if src is None or dst is None:
        real_n = int(np.prod(pa.size_local(pr))) * ncols * 8
        cplx_n = int(np.prod(pa.size_local(pc))) * ncols * 16
        a, b = HostBuf(real_n if flags == FWD else cplx_n), HostBuf(cplx_n if flags == FWD else real_n)
        call.keep = (a, b)
        src, dst = a.at(), b.at()
    n_extra = len(extra) if n_extra is None else n_extra
    return lib.pa_rfft(pr._h, pc._h, n_extra, i64arr(extra) if extra_ptr else None, flags, src, dst,
                       None)


def no_gpu():
    return lib.pa_device_count() == 0


@pytest.mark.parametrize("flags", [FWD, BWD])
@pytest.mark.parametrize("kw", [dict(), dict(perm=(1, 3, 2)), dict(real_dims=(2048, 3, 2)),
                                dict(real_dims=(6, 32, 4), perm=(2, 1, 3), decomp=(1, 3)),
                                dict(real_dims=(16, 0, 4))])
def test_valid_arguments_without_a_device_give_enogpu(flags, kw):
    if not no_gpu():
        pytest.skip("GPU present")
    pr, pc = pencils(**kw)
    assert call(pr, pc, flags) == _lib.PA_ENOGPU
    assert call(pr, pc, flags, extra=(2,)) == _lib.PA_ENOGPU


def test_empty_local_array_accepts_null_pointers():
    if not no_gpu():
        pytest.skip("GPU present")
    pr, pc = pencils(real_dims=(16, 0, 4))
    assert lib.pa_rfft(pr._h, pc._h, 0, None, FWD, None, None, None) == _lib.PA_ENOGPU


def test_incompatible_pencils():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    other = pa.MPITopology(pa.COMM_SELF, (1, 1))
    cases = [
        dict(topo=topo, ctopo=other),                                   # not the same topology object
        dict(real_dims=(16, 6, 4, 2), decomp=(2, 3), cdecomp=(2, 4)),   # different decomposition
        dict(cperm=(1, 3, 2)),                                          # different permutation
        dict(decomp=(1, 3)),                                            # transform axis decomposed
        dict(perm=(2, 1, 3), decomp=(2, 3)),                            # ... logical dim 2 (perm[1])
        dict(cplx_dims=(9, 6, 5)),                                      # other sizes differ
        dict(cplx_dims=(8, 6, 4)),                                      # not N/2+1
        dict(cplx_dims=(16, 6, 4)),
    ]
    for kw in cases:
        pr, pc = pencils(**kw)
        for flags in (FWD, BWD):
            assert call(pr, pc, flags) == _lib.PA_EINCOMPAT, kw
            assert lib.pa_last_error().startswith(b"pa_rfft")


def test_bad_flags():
    pr, pc = pencils()
    for flags in (0, FWD | BWD, FWD | _lib.PA_WAITALL, BWD | _lib.PA_NO_OVERLAP, 1):
        assert call(pr, pc, flags) == _lib.PA_EINVAL, flags
        assert b"flags" in lib.pa_last_error()


@pytest.mark.parametrize("n", [8, 24, 4096, 2])
def test_line_length_not_a_power_of_two_in_16_to_2048(n):
    pr, pc = pencils(real_dims=(n, 4, 4))
    assert call(pr, pc, FWD) == _lib.PA_EINVAL
    assert b"power of two" in lib.pa_last_error()


def test_null_pointers_for_non_empty_arrays():
    pr, pc = pencils()
    buf = HostBuf(16 * 9 * 24)
    for src, dst in ((None, buf.at()), (buf.at(), None), (None, None)):
        assert lib.pa_rfft(pr._h, pc._h, 0, None, FWD, src, dst, None) == _lib.PA_EINVAL
        assert b"null" in lib.pa_last_error()


def test_overlap_and_alignment():
    pr, pc = pencils()
    real_b, cplx_b = 16 * 24 * 8, 9 * 24 * 16
    buf = HostBuf(real_b + cplx_b + 64)
    for flags, nsrc, ndst in ((FWD, real_b, cplx_b), (BWD, cplx_b, real_b)):
        # overlapping by one 16-byte element either way, and fully aliased
        for s, d in ((0, nsrc - 16), (ndst - 16, 0), (0, 0)):
            assert call(pr, pc, flags, src=buf.at(s), dst=buf.at(d)) == _lib.PA_EINVAL, (flags, s, d)
            assert b"overlap" in lib.pa_last_error()
        # adjacent is fine (ENOGPU / OK past the checks); misaligned by 8 bytes is not
        for s, d in ((8, nsrc + 16), (0, nsrc + 8)):
            assert call(pr, pc, flags, src=buf.at(s), dst=buf.at(d)) == _lib.PA_EINVAL
            assert b"aligned" in lib.pa_last_error()
        if no_gpu():
            assert call(pr, pc, flags, src=buf.at(0), dst=buf.at(nsrc)) == _lib.PA_ENOGPU


def test_extra_dims_limits():
    pr, pc = pencils()
    if no_gpu():
        assert call(pr, pc, FWD, extra=(1, 1, 1, 1, 2)) == _lib.PA_ENOGPU    # 3 + 5 = PA_MAX_DIMS
    assert call(pr, pc, FWD, extra=(1, 1, 1, 1, 1, 2)) == _lib.PA_EINVAL     # 3 + 6 > PA_MAX_DIMS
    assert call(pr, pc, FWD, extra=(2,), extra_ptr=False) == _lib.PA_EINVAL  # NULL extra_dims
    assert call(pr, pc, FWD, extra=(2,), n_extra=-1) == _lib.PA_EINVAL
    buf = HostBuf(1 << 14)
    assert call(pr, pc, FWD, extra=(-2,), src=buf.at(0), dst=buf.at(1 << 13)) == _lib.PA_EINVAL


def test_python_wrappers_check_dtypes_and_extra_dims():
    """The dtype / extra-dims checks of rfft_ / brfft_ run before anything touches a device
    (CPU tensors stand in for the parent arrays here)."""
    pr, pc = pencils()

    def arr(p, dtype, *extra):
        mem = pa.size_local(p, pa.MemoryOrder())
        return pa.PencilArray(p, torch.zeros(tuple(reversed(mem + extra)), dtype=dtype), extra)

    xr, xc = arr(pr, torch.float64), arr(pc, torch.complex128)
    with pytest.raises(pa.ArgumentError):
        pa.rfft_(arr(pc, torch.complex64), xr)
    with pytest.raises(pa.ArgumentError):
        pa.rfft_(xc, arr(pr, torch.float32))
    with pytest.raises(pa.ArgumentError):
        pa.rfft_(xr, xc)                         # directions swapped
    with pytest.raises(pa.ArgumentError):
        pa.brfft_(xc, xr)
    with pytest.raises(pa.ArgumentError):
        pa.brfft_(arr(pr, torch.float32), xc)
    with pytest.raises(pa.ArgumentError):
        pa.rfft_(arr(pc, torch.complex128, 2), arr(pr, torch.float64, 3))
    with pytest.raises(pa.ArgumentError):
        pa.brfft_(arr(pr, torch.float64), arr(pc, torch.complex128, 2))
