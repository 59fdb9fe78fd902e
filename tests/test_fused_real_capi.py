"""`pa_transpose_r2r` / `pa_transpose_rfft` / `pa_plan_real_check` on the host (CPU): the fused
transposition of real arrays + DCT / DST or real-to-complex transform.

The verdict must be the same on every rank of a grid line (a rank that refused while its peers
went ahead would leave them waiting on the exchange), so real x -> y plans are built for every
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
KINDS = (_lib.PA_REDFT10, _lib.PA_REDFT01, _lib.PA_RODFT10, _lib.PA_RODFT01)


def no_gpu():
    return lib.pa_device_count() == 0


def real_xy(topo, dims, xperm=None, yperm=(2, 1, 3)):
    """Real x-pencil, real y-pencil and the complex y-pencil (N/2+1 along y) of a wall-bounded
    chain: the x -> y plan transposes the real arrays, the transform runs along y."""
    M = len(topo.dims)
    xdec, ydec = ((2, 3), (1, 3)) if M == 2 else ((2,), (1,))
    px = pa.Pencil(topo, dims, xdec, permute=pa.Permutation(*xperm) if xperm else None)
    py = pa.Pencil(px, decomp_dims=ydec, permute=pa.Permutation(*yperm) if yperm else pa.NoPermutation())
    ay = (yperm or (1, 2, 3))[0] - 1
    pyc = pa.Pencil(py, size_global=tuple(n // 2 + 1 if d == ay else n for d, n in enumerate(dims)))
    return px, py, pyc


def verdicts(grid, dims, extra=(), xperm=None, yperm=(2, 1, 3), f32=False):
    """{line (world ranks): {rank: status}} of the real x -> y plan on every emulated rank."""
    lines = {}
    for er in make_ranks(grid):
        px, py, _ = real_xy(er.topo, dims, xperm, yperm)
        plan = _Plan(px, py, extra, 4 if f32 else 8, pa.PointToPoint())
        st = lib.pa_plan_real_check(plan.h, F32 if f32 else 0)
        assert lib.pa_plan_real_check(plan.h, F32 if f32 else 0) == st  # cached: the same again
        info = plan.info
        line = tuple(sorted(plan.peer(n).world_rank for n in range(1, info.nproc + 1))) \
            if info.dim else (er.comm.rank,)
        lines.setdefault(line, {})[er.comm.rank] = st
    return lines


NS = [16, 32, 64, 128, 256, 512, 1024, 2048, 8, 24, 4096]
GRIDS = [(1, 1), (2, 1), (3, 2), (5, 1), (8, 1), (9, 1), (4,), (7,), (9,)]
SHAPES = [dict(), dict(xperm=(1, 3, 2)), dict(yperm=(2, 3, 1)), dict(yperm=None),
          dict(extra=(2,)), dict(extra=(1, 1, 1, 1, 2))]


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "x".join(map(str, g)))
def test_real_check_is_uniform_over_each_grid_line(grid):
    seen = set()
    for N, kw in itertools.product(NS, SHAPES):
        # few points along x and z: ranks that own nothing once 9 ranks split them
        dims = (3, N, 5) if N <= 512 else (2, N, 3)
        for f32 in (False, True):
            for line, per_rank in verdicts(grid, dims, f32=f32, **kw).items():
                got = set(per_rank.values())
                assert set(per_rank) == set(line), (grid, N, kw, line)
                assert len(got) == 1, (grid, N, kw, f32, per_rank)
                assert got <= {OK, EINVAL}
                seen |= got
                nproc = len(line)
                if N in (8, 24, 4096) or nproc > 8:
                    assert got == {EINVAL}, (grid, N, kw, f32)
    assert seen == ({EINVAL} if grid[0] > 8 else {OK, EINVAL})


@pytest.mark.parametrize("nproc,N,why", [(9, 32, "more than 8 blocks"), (3, 24, "power of two"),
                                         (1, 4096, "power of two"), (2, 8, "power of two")])
def test_real_check_reasons(nproc, N, why):
    for er in make_ranks((nproc,)):
        px, py, _ = real_xy(er.topo, (10, N, 3))
        plan = _Plan(px, py, (), 8, pa.PointToPoint())
        assert lib.pa_plan_real_check(plan.h, 0) == EINVAL
        assert why in lib.pa_last_error().decode()
    assert lib.pa_plan_real_check(None, 0) == EINVAL


def test_odd_block_boundaries_are_accepted():
    """N = 32 over 3 ranks: blocks of 11, 11 and 10 reals along the line, so complex slots are
    filled from two blocks.  Fusable on every rank."""
    for er in make_ranks((3,)):
        px, py, _ = real_xy(er.topo, (12, 32, 4))
        plan = _Plan(px, py, (), 8, pa.PointToPoint())
        assert lib.pa_plan_real_check(plan.h, 0) == OK
        assert lib.pa_plan_real_check(plan.h, F32) == EINVAL  # Float64 plan


def test_element_size_must_match_the_precision():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px, py, _ = real_xy(topo, (4, 64, 4))
    p8 = _Plan(px, py, (), 8, pa.PointToPoint())
    p4 = _Plan(px, py, (), 4, pa.PointToPoint())
    p16 = _Plan(px, py, (), 16, pa.PointToPoint())
    assert lib.pa_plan_real_check(p8.h, 0) == OK
    assert lib.pa_plan_real_check(p8.h, F32) == EINVAL
    assert lib.pa_plan_real_check(p4.h, F32) == OK
    assert lib.pa_plan_real_check(p4.h, 0) == EINVAL
    assert lib.pa_plan_real_check(p16.h, 0) == EINVAL
    assert lib.pa_plan_real_check(p16.h, F32) == EINVAL


@pytest.mark.parametrize("method", [pa.PeerPut(), pa.PeerGet()])
def test_one_sided_methods_are_refused_on_an_exchange(method):
    """PeerPut / PeerGet have no unpack pass to fuse with: refused by the check on every rank of
    a 2-rank line, and by Transposition(..., r2r= / rfft=) before any window registration.  A
    one-rank plan has no exchange, so there the method does not matter."""
    def arr(p, dtype):
        mem = pa.size_local(p, pa.MemoryOrder())
        return pa.PencilArray(p, torch.zeros(tuple(reversed(mem)), dtype=dtype))

    for er in make_ranks((2,)):
        px, py, pyc = real_xy(er.topo, (4, 32, 3))
        plan = _Plan(px, py, (), 8, method)
        assert lib.pa_plan_real_check(plan.h, 0) == EINVAL
        assert "one-sided" in lib.pa_last_error().decode()
        staged = _Plan(px, py, (), 8, pa.PointToPoint())
        assert lib.pa_plan_real_check(staged.h, 0) == OK
        with pytest.raises(pa.ArgumentError, match="one-sided"):
            pa.Transposition(arr(py, torch.float64), arr(px, torch.float64), method=method,
                             r2r="REDFT10")
        with pytest.raises(pa.ArgumentError, match="one-sided"):
            pa.Transposition(arr(pyc, torch.complex128), arr(px, torch.float64), method=method,
                             rfft=True)
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px, py, _ = real_xy(topo, (4, 32, 3))
    one = _Plan(px, py, (), 8, method)
    assert lib.pa_plan_real_check(one.h, 0) == OK


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("order", ["real_first", "fft_first", "brfft_first"])
def test_real_verdicts_are_cached_apart(f32, order):
    """An 8-byte plan is a ComplexF32 plan to pa_plan_fft_check_ex / pa_plan_brfft_check and a
    Float64 plan to pa_plan_real_check.  Lines of 16 elements: fusable as a complex FFT of 16
    points and as a real transform of N = 16, not as N/2+1 = 16 bins (no power-of-two N); lines
    of 9: only as 9 bins of N = 16.  No cached verdict answers for another, in any call order."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    es, flag = (4, F32) if f32 else (8, 0)
    for M, want_real, want_fft, want_brfft in ((16, OK, OK, EINVAL), (9, EINVAL, EINVAL, OK)):
        px = pa.Pencil(topo, (6, M, 4), (2, 3))
        py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
        plan = _Plan(px, py, (), es, pa.PointToPoint())
        # an 8-byte plan is ComplexF32 to the complex checks: they need PA_FFT_F32; a 4-byte
        # plan is nothing to them
        cflag = F32
        cwant_fft, cwant_brfft = (want_fft, want_brfft) if not f32 else (EINVAL, EINVAL)
        calls = {"real": lambda: lib.pa_plan_real_check(plan.h, flag) == want_real,
                 "fft": lambda: lib.pa_plan_fft_check_ex(plan.h, cflag) == cwant_fft,
                 "brfft": lambda: lib.pa_plan_brfft_check(plan.h, cflag) == cwant_brfft}
        first = order.split("_")[0]
        seq = [first] + [k for k in calls if k != first]
        for _ in range(2):
            for k in seq:
                assert calls[k](), (M, k)
        # the other precision is a verdict of its own (element size mismatch)
        assert lib.pa_plan_real_check(plan.h, flag ^ F32) == EINVAL


# ---- the ABI on host buffers ---------------------------------------------------------------
class HostBuf:
    """16-byte-aligned host memory (the checks only look at addresses and sizes)."""

    def __init__(self, nbytes):
        self.raw = np.zeros(nbytes + 64, dtype=np.uint8)
        a = self.raw.ctypes.data
        self.addr = a + (-a) % 16

    def at(self, off=0):
        return C.c_void_p(self.addr + off)


def setup(dims=(6, 32, 4), f32=False, extra=(), xperm=None):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px, py, pyc = real_xy(topo, dims, xperm)
    plan = _Plan(px, py, extra, 4 if f32 else 8, pa.PointToPoint())
    n = int(np.prod(extra)) if extra else 1
    rs = 4 if f32 else 8
    src_b = int(np.prod(pa.size_local(px))) * n * rs
    r2r_b = int(np.prod(pa.size_local(py))) * n * rs
    rfft_b = int(np.prod(pa.size_local(pyc))) * n * 2 * rs
    return topo, px, py, pyc, plan, src_b, r2r_b, rfft_b


def r2r(plan, kind, src, dst, flags=0):
    return lib.pa_transpose_r2r(plan.h, None, kind, src, dst, flags, None)


def rfft(plan, cplx, src, dst, flags=0):
    return lib.pa_transpose_rfft(plan.h, None, cplx._h, src, dst, flags, None)


VALID = [dict(), dict(f32=True), dict(dims=(3, 2048, 2)), dict(dims=(5, 16, 3)),
         dict(xperm=(1, 3, 2)), dict(extra=(2, 3))]


@pytest.mark.parametrize("kw", VALID)
def test_valid_arguments_without_a_device_give_enogpu(kw):
    if not no_gpu():
        pytest.skip("GPU present")
    _, _, _, pyc, plan, src_b, r2r_b, rfft_b = setup(**kw)
    buf = HostBuf(src_b + max(r2r_b, rfft_b))
    f = F32 if kw.get("f32") else 0
    for extra_flags in (0, _lib.PA_WAITALL, _lib.PA_NO_OVERLAP | _lib.PA_STAGE_SELF):
        for kind in KINDS:
            assert r2r(plan, kind, buf.at(0), buf.at(src_b), f | extra_flags) == ENOGPU
        assert rfft(plan, pyc, buf.at(0), buf.at(src_b), f | extra_flags) == ENOGPU


def test_empty_local_array_accepts_null_pointers():
    if not no_gpu():
        pytest.skip("GPU present")
    _, _, _, pyc, plan, src_b, r2r_b, rfft_b = setup(dims=(6, 32, 0))
    assert src_b == r2r_b == rfft_b == 0
    assert r2r(plan, _lib.PA_REDFT10, None, None) == ENOGPU
    assert rfft(plan, pyc, None, None) == ENOGPU


def test_bad_kinds():
    _, _, _, _, plan, src_b, r2r_b, _ = setup()
    buf = HostBuf(src_b + r2r_b)
    for kind in (0, 1, 2, 3, 6, 7, 10, -1):
        assert r2r(plan, kind, buf.at(0), buf.at(src_b)) == EINVAL, kind
        assert b"kind" in lib.pa_last_error()


def test_bad_flags():
    _, _, _, pyc, plan, src_b, r2r_b, rfft_b = setup()
    buf = HostBuf(src_b + max(r2r_b, rfft_b))
    for flags in (_lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD, _lib.PA_FFT_FORWARD | _lib.PA_WAITALL,
                  64, 1 << 31):
        assert r2r(plan, _lib.PA_REDFT10, buf.at(0), buf.at(src_b), flags) == EINVAL, flags
        assert b"flags" in lib.pa_last_error()
        assert rfft(plan, pyc, buf.at(0), buf.at(src_b), flags) == EINVAL, flags
        assert b"flags" in lib.pa_last_error()


def test_element_size_and_precision_mismatch():
    _, _, _, pyc, plan, src_b, r2r_b, rfft_b = setup()            # Float64 plan
    buf = HostBuf(src_b + max(r2r_b, rfft_b))
    assert r2r(plan, _lib.PA_REDFT01, buf.at(0), buf.at(src_b), F32) == EINVAL
    assert b"elsize" in lib.pa_last_error()
    assert rfft(plan, pyc, buf.at(0), buf.at(src_b), F32) == EINVAL
    assert b"elsize" in lib.pa_last_error()
    _, _, _, pyc, plan, src_b, r2r_b, rfft_b = setup(f32=True)    # Float32 plan
    assert r2r(plan, _lib.PA_REDFT01, buf.at(0), buf.at(src_b), 0) == EINVAL
    assert b"elsize" in lib.pa_last_error()
    assert rfft(plan, pyc, buf.at(0), buf.at(src_b), 0) == EINVAL
    assert b"elsize" in lib.pa_last_error()
    # a complex (elsize 16) plan is not a real plan in either precision
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px, py, pyc = real_xy(topo, (6, 32, 4))
    p16 = _Plan(px, py, (), 16, pa.PointToPoint())
    for f in (0, F32):
        assert r2r(p16, _lib.PA_REDFT10, buf.at(0), buf.at(1 << 12), f) == EINVAL
        assert rfft(p16, pyc, buf.at(0), buf.at(1 << 12), f) == EINVAL


def test_unrelated_complex_pencils():
    topo, px, py, pyc, plan, src_b, _, rfft_b = setup()
    buf = HostBuf(1 << 16)
    other = pa.MPITopology(pa.COMM_SELF, (1, 1))
    wrong = [
        pa.Pencil(other, (6, 17, 4), (1, 3), permute=pa.Permutation(2, 1, 3)),  # another topology
        pa.Pencil(pyc, size_global=(6, 16, 4)),                               # not N/2+1 = 17 bins
        pa.Pencil(pyc, size_global=(6, 18, 4)),
        pa.Pencil(pyc, decomp_dims=(2, 3)),                                   # other decomposition
        pa.Pencil(pyc, permute=pa.Permutation(2, 3, 1)),                      # other permutation
        pa.Pencil(pyc, permute=pa.NoPermutation()),
        pa.Pencil(pyc, size_global=(6, 17, 5)),                               # other sizes differ
    ]
    for cplx in wrong:
        assert rfft(plan, cplx, buf.at(0), buf.at(1 << 15)) == EINCOMPAT
        assert lib.pa_last_error().startswith(b"pa_transpose_rfft")
    # the matching pencil runs: on device arrays when there is a GPU (a kernel cannot address
    # this host memory)
    if no_gpu():
        assert rfft(plan, pyc, buf.at(0), buf.at(1 << 15)) == ENOGPU
    else:
        src = torch.zeros(src_b, dtype=torch.uint8, device="cuda")
        dst = torch.empty(rfft_b, dtype=torch.uint8, device="cuda")
        assert rfft(plan, pyc, C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr())) == OK
        torch.cuda.synchronize()
    assert lib.pa_transpose_rfft(plan.h, None, None, buf.at(0), buf.at(1 << 15), 0, None) == EINVAL
    # a plan whose output axis is decomposed (y -> x with the rfft along y): no match either
    back = _Plan(py, px, (), 8, pa.PointToPoint())
    assert rfft(back, pyc, buf.at(0), buf.at(1 << 15)) == EINCOMPAT


def test_decomposed_transform_axis():
    """The transform runs along the output pencil's first memory dim, which must not be
    decomposed (as for r2r_ / rfft_), even over one rank: refused before the geometry check."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (32, 6, 4), (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3))            # first memory dim x, decomposed
    pyc = pa.Pencil(py, size_global=(17, 6, 4))
    plan = _Plan(px, py, (), 8, pa.PointToPoint())
    buf = HostBuf(1 << 14)
    assert r2r(plan, _lib.PA_REDFT10, buf.at(0), buf.at(1 << 13)) == EINCOMPAT
    assert b"decomposed" in lib.pa_last_error()
    assert rfft(plan, pyc, buf.at(0), buf.at(1 << 13)) == EINCOMPAT
    assert b"decomposed" in lib.pa_last_error()


def test_line_length_refused_by_the_check():
    for dims in ((4, 24, 4), (4, 8, 4), (2, 4096, 2)):
        _, _, _, pyc, plan, src_b, r2r_b, rfft_b = setup(dims=dims)
        buf = HostBuf(src_b + max(r2r_b, rfft_b))
        assert r2r(plan, _lib.PA_REDFT10, buf.at(0), buf.at(src_b)) == EINVAL
        assert b"power of two" in lib.pa_last_error()
        assert rfft(plan, pyc, buf.at(0), buf.at(src_b)) == EINVAL
        assert b"power of two" in lib.pa_last_error()


@pytest.mark.parametrize("which", ["r2r", "rfft"])
def test_null_pointers_overlap_and_alignment(which):
    _, _, _, pyc, plan, src_b, r2r_b, rfft_b = setup()
    dst_b = r2r_b if which == "r2r" else rfft_b
    buf = HostBuf(src_b + dst_b + 64)

    def call(s, d):
        return r2r(plan, _lib.PA_RODFT01, s, d) if which == "r2r" else rfft(plan, pyc, s, d)

    for s, d in ((None, buf.at(src_b)), (buf.at(0), None), (None, None)):
        assert call(s, d) == EINVAL
        assert b"null" in lib.pa_last_error()
    # overlapping by one element either way, and aliased
    for s, d in ((0, src_b - 16), (dst_b - 16, 0), (0, 0)):
        assert call(buf.at(s), buf.at(d)) == EINVAL, (s, d)
        assert b"overlap" in lib.pa_last_error()
    # dst only 8-byte aligned
    assert call(buf.at(0), buf.at(src_b + 8)) == EINVAL
    assert b"aligned" in lib.pa_last_error()
    if no_gpu():
        assert call(buf.at(0), buf.at(src_b)) == ENOGPU  # adjacent is fine
    assert lib.pa_transpose_r2r(None, None, _lib.PA_REDFT10, buf.at(0), buf.at(src_b), 0, None) == EINVAL
    assert lib.pa_transpose_rfft(None, None, pyc._h, buf.at(0), buf.at(src_b), 0, None) == EINVAL


def test_python_wrappers():
    """dtypes, kinds, exclusive modes and fft= on a fused real transposition are refused before
    any device work (CPU tensors stand in for the parent arrays)."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px, py, pyc = real_xy(topo, (6, 32, 4))

    def arr(p, dtype, *extra):
        mem = pa.size_local(p, pa.MemoryOrder())
        return pa.PencilArray(p, torch.zeros(tuple(reversed(mem + extra)), dtype=dtype), extra)

    for kind in ("DCT", "REDFT00", "redft10", 5, ""):
        with pytest.raises(pa.ArgumentError):
            pa.Transposition(arr(py, torch.float64), arr(px, torch.float64), r2r=kind)
    for od, idt in ((torch.float32, torch.float64), (torch.complex128, torch.complex128),
                    (torch.float16, torch.float16)):
        with pytest.raises(pa.ArgumentError):
            pa.Transposition(arr(py, od), arr(px, idt), r2r="REDFT10")
    for cd, rd in ((torch.complex128, torch.float32), (torch.complex64, torch.float64),
                   (torch.float64, torch.float64), (torch.complex128, torch.complex128)):
        with pytest.raises(pa.ArgumentError):
            pa.Transposition(arr(pyc, cd), arr(px, rd), rfft=True)
    with pytest.raises(pa.ArgumentError, match="exclude"):
        pa.Transposition(arr(pyc, torch.complex128), arr(px, torch.float64), rfft=True, r2r="REDFT10")
    with pytest.raises(pa.ArgumentError, match="exclude"):
        pa.Transposition(arr(py, torch.float64), arr(px, torch.float64), brfft=True, r2r="REDFT10")
    with pytest.raises(pa.ArgumentError, match="exclude"):
        pa.Transposition(arr(pyc, torch.complex128), arr(px, torch.float64), brfft=True, rfft=True)
    with pytest.raises(pa.ArgumentError):
        pa.Transposition(arr(py, torch.float64, 2), arr(px, torch.float64, 3), r2r="REDFT10")

    t = pa.Transposition(arr(py, torch.float64), arr(px, torch.float64), r2r="REDFT10")
    assert t.fft_fusable() and t.Po is py
    tr = pa.Transposition(arr(pyc, torch.complex128), arr(px, torch.float64), rfft=True)
    assert tr.Po.size_global == (6, 32, 4) and tr.Po.perm == py.perm
    tr2 = pa.Transposition(arr(pyc, torch.complex128), arr(px, torch.float64), rfft=True)
    assert tr2.Po is tr.Po and tr2.plan is tr.plan  # one derived pencil, one plan
    assert tr.fft_fusable()
    for tt in (t, tr):
        for fft in ("backward", "forward"):
            with pytest.raises(pa.ArgumentError):
                pa.transpose_(tt, fft=fft)
    t32 = pa.Transposition(arr(py, torch.float32), arr(px, torch.float32), r2r="RODFT01")
    assert t32.fft_fusable()
    tr32 = pa.Transposition(arr(pyc, torch.complex64), arr(px, torch.float32), rfft=True)
    assert tr32.fft_fusable()
    # N = 24 is planned, but not fusable
    px24, py24, _ = real_xy(topo, (6, 24, 4))
    t24 = pa.Transposition(arr(py24, torch.float64), arr(px24, torch.float64), r2r="REDFT10")
    assert not t24.fft_fusable()
