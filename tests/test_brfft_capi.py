"""`pa_transpose_brfft` / `pa_plan_brfft_check` on the host (CPU): the fused y->x transpose +
complex-to-real transform of a real-input backward FFT.

The verdict must be the same on every rank of a grid line (a rank that refused while its peers
went ahead would leave them waiting on the exchange), so real-input chains are planned for every
emulated rank and the ranks of each line compared.  The ABI refuses bad arguments before any
device call; valid arguments without a device give PA_ENOGPU."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib
from pencilarrays_b200.transpositions import _Plan
from util import make_ranks

OK, EINVAL, EINCOMPAT, ENOGPU = _lib.PA_OK, _lib.PA_EINVAL, _lib.PA_EINCOMPAT, _lib.PA_ENOGPU
F32 = _lib.PA_FFT_F32


def no_gpu():
    return lib.pa_device_count() == 0


def real_chain(topo, dims, xperm=None, yperm=(2, 1, 3)):
    """Real x-pencil, its complex counterpart and the complex y-pencil of a real-input plan."""
    M = len(topo.dims)
    xdec, ydec = ((2, 3), (1, 3)) if M == 2 else ((2,), (1,))
    pxr = pa.Pencil(topo, dims, xdec, permute=pa.Permutation(*xperm) if xperm else None)
    ax = (xperm or (1, 2, 3))[0] - 1
    pxc = pa.Pencil(pxr, size_global=tuple(n // 2 + 1 if d == ax else n for d, n in enumerate(dims)))
    pyc = pa.Pencil(pxc, decomp_dims=ydec, permute=pa.Permutation(*yperm) if yperm else pa.NoPermutation())
    return pxr, pxc, pyc


def verdicts(grid, dims, extra=(), xperm=None, yperm=(2, 1, 3), f32=False):
    """{line (world ranks): {rank: status}} of the y -> x plan on every emulated rank."""
    lines = {}
    for er in make_ranks(grid):
        _, pxc, pyc = real_chain(er.topo, dims, xperm, yperm)
        plan = _Plan(pyc, pxc, extra, 8 if f32 else 16, pa.PointToPoint())
        st = lib.pa_plan_brfft_check(plan.h, F32 if f32 else 0)
        assert lib.pa_plan_brfft_check(plan.h, F32 if f32 else 0) == st  # cached: the same again
        info = plan.info
        line = tuple(sorted(plan.peer(n).world_rank for n in range(1, info.nproc + 1))) \
            if info.dim else (er.comm.rank,)
        lines.setdefault(line, {})[er.comm.rank] = st
    return lines


NS = [16, 32, 64, 128, 256, 512, 1024, 2048, 24, 4096]
GRIDS = [(1, 1), (2, 1), (3, 2), (5, 1), (8, 1), (9, 1), (4,), (7,), (9,)]
SHAPES = [dict(), dict(xperm=(1, 3, 2)), dict(yperm=(2, 3, 1)), dict(yperm=None),
          dict(extra=(2,)), dict(extra=(1, 1, 1, 1, 2))]


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "x".join(map(str, g)))
def test_brfft_check_is_uniform_over_each_grid_line(grid):
    seen = set()
    for N, kw in itertools.product(NS, SHAPES):
        # few points along y and z: ranks that own nothing once 9 ranks split them
        dims = (N, 3, 5) if N <= 512 else (N, 2, 3)
        for f32 in (False, True):
            for line, per_rank in verdicts(grid, dims, f32=f32, **kw).items():
                got = set(per_rank.values())
                assert set(per_rank) == set(line), (grid, N, kw, line)
                assert len(got) == 1, (grid, N, kw, f32, per_rank)
                assert got <= {OK, EINVAL}
                seen |= got
                nproc = len(line)
                if N in (24, 4096) or nproc > 8:
                    assert got == {EINVAL}, (grid, N, kw, f32)
    assert seen == ({EINVAL} if grid[0] > 8 else {OK, EINVAL})


@pytest.mark.parametrize("nproc,N,why", [(9, 32, "more than 8 blocks"), (3, 24, "N/2+1"),
                                         (1, 4096, "N/2+1"), (2, 8, "N/2+1")])
def test_brfft_check_reasons(nproc, N, why):
    for er in make_ranks((nproc,)):
        _, pxc, pyc = real_chain(er.topo, (N, 10, 3))
        plan = _Plan(pyc, pxc, (), 16, pa.PointToPoint())
        assert lib.pa_plan_brfft_check(plan.h, 0) == EINVAL
        assert why in lib.pa_last_error().decode()
    assert lib.pa_plan_brfft_check(None, 0) == EINVAL


def test_element_size_must_match_the_precision():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    _, pxc, pyc = real_chain(topo, (64, 4, 4))
    # (the plans stay referenced while their handles are in use)
    p16 = _Plan(pyc, pxc, (), 16, pa.PointToPoint())
    p8 = _Plan(pyc, pxc, (), 8, pa.PointToPoint())
    assert lib.pa_plan_brfft_check(p16.h, 0) == OK
    assert lib.pa_plan_brfft_check(p16.h, F32) == EINVAL
    assert lib.pa_plan_brfft_check(p8.h, F32) == OK
    assert lib.pa_plan_brfft_check(p8.h, 0) == EINVAL


@pytest.mark.parametrize("method", [pa.PeerPut(), pa.PeerGet()])
def test_one_sided_methods_are_refused_on_an_exchange(method):
    """PeerPut / PeerGet have no unpack pass to fuse with: refused by the check on every rank of
    a 2-rank line, and by Transposition(..., brfft=True) before any window registration.  A
    one-rank plan has no exchange, so there the method does not matter."""
    for er in make_ranks((2,)):
        pxr, pxc, pyc = real_chain(er.topo, (32, 4, 3))
        plan = _Plan(pyc, pxc, (), 16, method)
        assert lib.pa_plan_brfft_check(plan.h, 0) == EINVAL
        assert "one-sided" in lib.pa_last_error().decode()
        staged = _Plan(pyc, pxc, (), 16, pa.PointToPoint())
        assert lib.pa_plan_brfft_check(staged.h, 0) == OK

        def arr(p, dtype):
            mem = pa.size_local(p, pa.MemoryOrder())
            return pa.PencilArray(p, torch.zeros(tuple(reversed(mem)), dtype=dtype))

        with pytest.raises(pa.ArgumentError, match="one-sided"):
            pa.Transposition(arr(pxr, torch.float64), arr(pyc, torch.complex128), method=method,
                             brfft=True)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    _, pxc, pyc = real_chain(topo, (32, 4, 3))
    one = _Plan(pyc, pxc, (), 16, method)
    assert lib.pa_plan_brfft_check(one.h, 0) == OK


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("brfft_first", [False, True])
def test_brfft_and_fft_verdicts_are_cached_apart(f32, brfft_first):
    """A y -> x plan whose lines are 9 bins (N = 16) is fusable with brfft, not with a complex
    FFT; one of 16 bins (N = 30) the other way round.  Neither cached verdict answers for the
    other, whichever is asked first."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    es, flag = (8, F32) if f32 else (16, 0)
    for M, want_brfft, want_fft in ((9, OK, EINVAL), (16, EINVAL, OK)):
        px = pa.Pencil(topo, (M, 6, 4), (2, 3))
        py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        plan = _Plan(py, px, (), es, pa.PointToPoint())
        for _ in range(2):
            if brfft_first:
                assert lib.pa_plan_brfft_check(plan.h, flag) == want_brfft, M
                assert lib.pa_plan_fft_check_ex(plan.h, flag) == want_fft, M
            else:
                assert lib.pa_plan_fft_check_ex(plan.h, flag) == want_fft, M
                assert lib.pa_plan_brfft_check(plan.h, flag) == want_brfft, M
        # the other precision is a verdict of its own (element size mismatch)
        assert lib.pa_plan_brfft_check(plan.h, flag ^ F32) == EINVAL


# ---- the ABI on host buffers ---------------------------------------------------------------
class HostBuf:
    """16-byte-aligned host memory (the checks only look at addresses and sizes)."""

    def __init__(self, nbytes):
        self.raw = np.zeros(nbytes + 64, dtype=np.uint8)
        a = self.raw.ctypes.data
        self.addr = a + (-a) % 16

    def at(self, off=0):
        return C.c_void_p(self.addr + off)


def setup(dims=(32, 6, 4), f32=False, extra=(), xperm=None):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pxr, pxc, pyc = real_chain(topo, dims, xperm)
    plan = _Plan(pyc, pxc, extra, 8 if f32 else 16, pa.PointToPoint())
    n = int(np.prod(extra)) if extra else 1
    rs = 4 if f32 else 8
    src_b = int(np.prod(pa.size_local(pyc))) * n * 2 * rs
    dst_b = int(np.prod(pa.size_local(pxr))) * n * rs
    return topo, pxr, pxc, pyc, plan, src_b, dst_b


def call(plan, real, src, dst, flags=0):
    return lib.pa_transpose_brfft(plan.h, None, real._h, src, dst, flags, None)


@pytest.mark.parametrize("kw", [dict(), dict(f32=True), dict(dims=(2048, 3, 2)), dict(dims=(16, 5, 3)),
                                dict(xperm=(1, 3, 2)), dict(extra=(2, 3))])
def test_valid_arguments_without_a_device_give_enogpu(kw):
    if not no_gpu():
        pytest.skip("GPU present")
    _, pxr, _, _, plan, src_b, dst_b = setup(**kw)
    buf = HostBuf(src_b + dst_b)
    f = F32 if kw.get("f32") else 0
    for extra_flags in (0, _lib.PA_WAITALL, _lib.PA_NO_OVERLAP | _lib.PA_STAGE_SELF):
        assert call(plan, pxr, buf.at(0), buf.at(src_b), f | extra_flags) == ENOGPU


def test_empty_local_array_accepts_null_pointers():
    if not no_gpu():
        pytest.skip("GPU present")
    _, pxr, _, _, plan, src_b, dst_b = setup(dims=(32, 0, 4))
    assert src_b == dst_b == 0
    assert call(plan, pxr, None, None) == ENOGPU


def test_bad_flags():
    _, pxr, _, _, plan, src_b, dst_b = setup()
    buf = HostBuf(src_b + dst_b)
    for flags in (_lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD, _lib.PA_FFT_BACKWARD | _lib.PA_WAITALL,
                  64, 1 << 31):
        assert call(plan, pxr, buf.at(0), buf.at(src_b), flags) == EINVAL, flags
        assert b"flags" in lib.pa_last_error()


def test_element_size_and_precision_mismatch():
    _, pxr, _, _, plan, src_b, dst_b = setup()            # ComplexF64 plan
    buf = HostBuf(src_b + dst_b)
    assert call(plan, pxr, buf.at(0), buf.at(src_b), F32) == EINVAL
    assert b"elsize" in lib.pa_last_error()
    _, pxr, _, _, plan, src_b, dst_b = setup(f32=True)    # ComplexF32 plan
    assert call(plan, pxr, buf.at(0), buf.at(src_b), 0) == EINVAL
    assert b"elsize" in lib.pa_last_error()


def test_pencil_mismatches():
    topo, pxr, pxc, pyc, plan, src_b, dst_b = setup()
    buf = HostBuf(1 << 16)
    other = pa.MPITopology(pa.COMM_SELF, (1, 1))
    wrong = [
        pa.Pencil(other, (32, 6, 4), (2, 3)),                                 # another topology object
        pa.Pencil(pxr, decomp_dims=(1, 3)),                                   # other decomposition
        pa.Pencil(pxr, permute=pa.Permutation(1, 3, 2)),                      # other permutation
        pa.Pencil(pxr, size_global=(30, 6, 4)),                               # not N/2+1 = 16 bins
        pa.Pencil(pxr, size_global=(32, 6, 5)),                               # other sizes differ
        pyc,                                                                  # the input pencil
    ]
    for real in wrong:
        assert call(plan, real, buf.at(0), buf.at(1 << 15)) == EINCOMPAT
        assert lib.pa_last_error().startswith(b"pa_transpose_brfft")
    # a plan whose output axis is decomposed (x -> y): the real pencil cannot match it
    py_plan = _Plan(pxc, pyc, (), 16, pa.PointToPoint())
    assert call(py_plan, pxr, buf.at(0), buf.at(1 << 15)) == EINCOMPAT


def test_line_length_refused_by_the_check():
    _, pxr, _, _, plan, src_b, dst_b = setup(dims=(24, 4, 4))
    buf = HostBuf(src_b + dst_b)
    assert call(plan, pxr, buf.at(0), buf.at(src_b)) == EINVAL
    assert b"power of two" in lib.pa_last_error()


def test_null_pointers_overlap_and_alignment():
    _, pxr, _, _, plan, src_b, dst_b = setup()
    buf = HostBuf(src_b + dst_b + 64)
    for s, d in ((None, buf.at(src_b)), (buf.at(0), None), (None, None)):
        assert call(plan, pxr, s, d) == EINVAL
        assert b"null" in lib.pa_last_error()
    # overlapping by one element either way, and aliased
    for s, d in ((0, src_b - 16), (dst_b - 16, 0), (0, 0)):
        assert call(plan, pxr, buf.at(s), buf.at(d)) == EINVAL, (s, d)
        assert b"overlap" in lib.pa_last_error()
    # dst only 8-byte aligned
    assert call(plan, pxr, buf.at(0), buf.at(src_b + 8)) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    if no_gpu():
        assert call(plan, pxr, buf.at(0), buf.at(src_b)) == ENOGPU  # adjacent is fine
    assert lib.pa_transpose_brfft(None, None, pxr._h, buf.at(0), buf.at(src_b), 0, None) == EINVAL
    assert lib.pa_transpose_brfft(plan.h, None, None, buf.at(0), buf.at(src_b), 0, None) == EINVAL


def test_python_wrappers():
    """dtype pairs, and fft= on a brfft transposition, are refused before any device work
    (CPU tensors stand in for the parent arrays)."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pxr, pxc, pyc = real_chain(topo, (32, 6, 4))

    def arr(p, dtype, *extra):
        mem = pa.size_local(p, pa.MemoryOrder())
        return pa.PencilArray(p, torch.zeros(tuple(reversed(mem + extra)), dtype=dtype), extra)

    for rd, cd in ((torch.float32, torch.complex128), (torch.float64, torch.complex64),
                   (torch.complex128, torch.complex128), (torch.float64, torch.float64)):
        with pytest.raises(pa.ArgumentError):
            pa.Transposition(arr(pxr, rd), arr(pyc, cd), brfft=True)
    with pytest.raises(pa.ArgumentError):
        pa.Transposition(arr(pxr, torch.float64, 2), arr(pyc, torch.complex128, 3), brfft=True)
    # without brfft=True mixed element types are refused as before
    with pytest.raises(pa.ArgumentError):
        pa.Transposition(arr(pxr, torch.float64), arr(pyc, torch.complex128))
    t = pa.Transposition(arr(pxr, torch.float64), arr(pyc, torch.complex128), brfft=True)
    assert t.Po.size_global == (17, 6, 4)
    t2 = pa.Transposition(arr(pxr, torch.float64), arr(pyc, torch.complex128), brfft=True)
    assert t2.Po is t.Po and t2.plan is t.plan  # one derived pencil, one plan
    assert t.fft_fusable()
    for fft in ("backward", "forward"):
        with pytest.raises(pa.ArgumentError):
            pa.transpose_(t, fft=fft)
    t32 = pa.Transposition(arr(pxr, torch.float32), arr(pyc, torch.complex64), brfft=True)
    assert t32.fft_fusable()
