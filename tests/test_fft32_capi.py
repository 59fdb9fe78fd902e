"""Single precision (PA_FFT_F32) at the C-ABI boundary, on the host: every refusal is decided
before any device call.

* `pa_plan_fft_check_ex`: the flag asks about ComplexF32 (elsize 8), its absence about
  ComplexF64 (elsize 16), and the element size alone never selects single precision; the verdict
  is the same on every rank of each grid line for every configuration of tests/test_fft_check.py,
  and each precision's cached verdict is independent of the other's, in both call orders;
* `pa_transpose` refuses a ComplexF32 fused FFT on an elsize-16 plan (and the bare flag);
* `pa_rfft` with the flag: line lengths, null / overlapping pointers sized with 4- and 8-byte
  elements, misalignment, and the Python wrappers' dtype pairs."""
import ctypes as C

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, i64arr
from pencilarrays_b200.transpositions import _Plan
import test_fft_check as fc
from util import build_chain

F32 = _lib.PA_FFT_F32
FWD, BWD = _lib.PA_FFT_FORWARD, _lib.PA_FFT_BACKWARD


def no_gpu():
    return lib.pa_device_count() == 0


def test_flag_value_is_distinct():
    assert F32 == 32
    assert F32 not in (_lib.PA_WAITALL, _lib.PA_NO_OVERLAP, _lib.PA_STAGE_SELF, FWD, BWD)


def _xy_plans(elsize):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (16, 8, 4), (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    return _Plan(px, py, (), elsize, pa.PointToPoint())


def test_check_ex_selects_the_precision_by_flag_only():
    p16, p8 = _xy_plans(16), _xy_plans(8)
    assert lib.pa_plan_fft_check_ex(p16.h, 0) == _lib.PA_OK
    assert lib.pa_plan_fft_check_ex(p16.h, F32) == _lib.PA_EINVAL
    assert b"8-byte" in lib.pa_last_error()
    assert lib.pa_plan_fft_check_ex(p8.h, F32) == _lib.PA_OK
    # elsize 8 without the flag: Float64, refused exactly as by pa_plan_fft_check
    assert lib.pa_plan_fft_check_ex(p8.h, 0) == _lib.PA_EINVAL
    assert b"ComplexF64 (16-byte) elements only" in lib.pa_last_error()
    assert lib.pa_plan_fft_check(p8.h) == _lib.PA_EINVAL
    # the other pa_transpose flags do not matter
    assert lib.pa_plan_fft_check_ex(p8.h, F32 | FWD | _lib.PA_WAITALL) == _lib.PA_OK
    assert lib.pa_plan_fft_check_ex(p16.h, FWD | _lib.PA_STAGE_SELF) == _lib.PA_OK
    assert lib.pa_plan_fft_check_ex(None, F32) == _lib.PA_EINVAL


@pytest.mark.parametrize("first", ["f64", "f32"])
def test_cached_verdicts_are_kept_per_precision(first):
    """An elsize-8 plan: ComplexF64 refused, ComplexF32 accepted; an elsize-16 plan the other way
    round.  Each answer, and its reason, survives asking the other precision in between."""
    p8, p16 = _xy_plans(8), _xy_plans(16)
    want = {(8, 0): (_lib.PA_EINVAL, b"16-byte"), (8, F32): (_lib.PA_OK, None),
            (16, 0): (_lib.PA_OK, None), (16, F32): (_lib.PA_EINVAL, b"8-byte")}
    order = [0, F32] if first == "f64" else [F32, 0]
    for _ in range(3):
        for flag in order:
            for es, p in ((8, p8), (16, p16)):
                st, why = want[(es, flag)]
                got = lib.pa_plan_fft_check_ex(p.h, flag) if flag else lib.pa_plan_fft_check(p.h)
                assert got == st, (first, es, flag)
                if why:
                    assert why in lib.pa_last_error(), (first, es, flag)


def _answers(case):
    """Per step: ({world rank: (ComplexF32 verdict on elsize 8, ComplexF64 on elsize 16)},
    {line: members})."""
    ranks, steps = build_chain(case)
    out = []
    for k in range(1, len(steps)):
        per_rank, lines = {}, {}
        for r in range(len(ranks)):
            a, b = steps[k - 1][r][0], steps[k][r][0]
            p8 = _Plan(a, b, case["extra"], 8, pa.PointToPoint())
            p16 = _Plan(a, b, case["extra"], 16, pa.PointToPoint())
            per_rank[r] = (lib.pa_plan_fft_check_ex(p8.h, F32), lib.pa_plan_fft_check(p16.h))
            info = p8.info
            line = tuple(sorted(p8.peer(n).world_rank for n in range(1, info.nproc + 1))) \
                if info.dim else (r,)
            lines.setdefault(line, set()).add(r)
        out.append((per_rank, lines))
    return out


@pytest.mark.parametrize("case", fc.RANDOM_CASES + fc.POW2_CASES,
                         ids=[c["name"] for c in fc.RANDOM_CASES + fc.POW2_CASES])
def test_check_ex_is_uniform_over_each_grid_line(case):
    """The 60 random and 40 power-of-two configurations: one ComplexF32 answer per grid line, and
    it is the ComplexF64 answer of the same geometry (the checks look at the blocks, not at the
    element size)."""
    for k, (per_rank, lines) in enumerate(_answers(case), start=1):
        for line, members in lines.items():
            assert members == set(line), (case["name"], k, line, members)
            got = {per_rank[r][0] for r in line}
            assert len(got) == 1, (case["name"], k, {r: per_rank[r] for r in line})
            assert got <= {_lib.PA_OK, _lib.PA_EINVAL}
            for r in line:
                assert per_rank[r][0] == per_rank[r][1], (case["name"], k, r, per_rank[r])


def test_seeded_configurations_see_both_answers():
    seen = {per_rank[r][0] for c in fc.POW2_CASES for per_rank, _ in _answers(c) for r in per_rank}
    assert seen == {_lib.PA_OK, _lib.PA_EINVAL}


@pytest.mark.parametrize("nproc,L,ok", [(3, 64, True), (8, 8, True), (6, 1024, True),
                                         (3, 48, False), (2, 2048, False), (9, 16, False)])
def test_check_ex_line_verdicts(nproc, L, ok):
    for r in range(nproc):
        topo = pa.MPITopology(pa.Comm(r, nproc), (nproc,))
        pa_ = pa.Pencil(topo, (L, nproc + 1, 3), (1,), permute=pa.Permutation(2, 1, 3))
        pb = pa.Pencil(pa_, decomp_dims=(2,), permute=pa.NoPermutation())
        p = _Plan(pa_, pb, (), 8, pa.PointToPoint())
        st = lib.pa_plan_fft_check_ex(p.h, F32)
        assert st == (_lib.PA_OK if ok else _lib.PA_EINVAL), (nproc, L, r)
        assert lib.pa_plan_fft_check_ex(p.h, F32) == st


class HostBuf:
    """16-byte-aligned host memory (the checks only look at addresses and sizes)."""

    def __init__(self, nbytes):
        self.raw = np.zeros(nbytes + 64, dtype=np.uint8)
        a = self.raw.ctypes.data
        self.addr = a + (-a) % 16

    def at(self, off=0):
        return C.c_void_p(self.addr + off)


def test_transpose_refuses_f32_on_a_16_byte_plan_before_any_device_call():
    p16 = _xy_plans(16)
    buf = HostBuf(2 * 16 * 16 * 8 * 4)
    n0 = lib.pa_launch_count()
    for d in (FWD, BWD):
        st = lib.pa_transpose(p16.h, None, buf.at(0), buf.at(16 * 16 * 8 * 4), d | F32 | _lib.PA_WAITALL,
                              None)
        assert st == _lib.PA_EINVAL and b"8-byte" in lib.pa_last_error()
    # the flag without a direction means nothing: refused
    p8 = _xy_plans(8)
    assert lib.pa_transpose(p8.h, None, buf.at(0), buf.at(16 * 16 * 8 * 4), F32, None) == _lib.PA_EINVAL
    assert b"PA_FFT_F32" in lib.pa_last_error()
    assert lib.pa_launch_count() == n0


# ---- pa_rfft with PA_FFT_F32 ----------------------------------------------------------------
def _pencils(real_dims=(16, 6, 4)):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pr = pa.Pencil(topo, real_dims, (2, 3))
    pc = pa.Pencil(pr, size_global=(real_dims[0] // 2 + 1,) + tuple(real_dims[1:]))
    return pr, pc


def _bytes(pr, pc):
    """(real, complex) bytes of the local arrays in single precision"""
    return (int(np.prod(pa.size_local(pr))) * 4, int(np.prod(pa.size_local(pc))) * 8)


@pytest.mark.parametrize("d", [FWD, BWD])
@pytest.mark.parametrize("dims", [(16, 6, 4), (2048, 3, 2), (32, 7, 1), (16, 0, 4)])
def test_rfft_f32_valid_arguments_without_a_device_give_enogpu(d, dims):
    if not no_gpu():
        pytest.skip("GPU present")
    pr, pc = _pencils(dims)
    rb, cb = _bytes(pr, pc)
    buf = HostBuf(rb + cb + 64)
    src, dst = (buf.at(0), buf.at(rb + 16 - rb % 16)) if d == FWD else (buf.at(0), buf.at(cb + 16 - cb % 16))
    assert lib.pa_rfft(pr._h, pc._h, 0, None, d | F32, src, dst, None) == _lib.PA_ENOGPU


def test_rfft_f32_flags():
    pr, pc = _pencils()
    buf = HostBuf(4096)
    for flags in (F32, FWD | BWD | F32, FWD | F32 | _lib.PA_WAITALL, BWD | F32 | _lib.PA_STAGE_SELF, F32 | 64):
        assert lib.pa_rfft(pr._h, pc._h, 0, None, flags, buf.at(0), buf.at(2048), None) == _lib.PA_EINVAL
        assert b"flags" in lib.pa_last_error()


@pytest.mark.parametrize("n", [8, 24, 4096, 2])
def test_rfft_f32_line_length(n):
    pr, pc = _pencils((n, 4, 4))
    buf = HostBuf(1 << 16)
    assert lib.pa_rfft(pr._h, pc._h, 0, None, FWD | F32, buf.at(0), buf.at(1 << 15), None) == _lib.PA_EINVAL
    assert b"power of two" in lib.pa_last_error()


def test_rfft_f32_null_pointers():
    pr, pc = _pencils()
    buf = HostBuf(4096)
    for src, dst in ((None, buf.at()), (buf.at(), None), (None, None)):
        assert lib.pa_rfft(pr._h, pc._h, 0, None, FWD | F32, src, dst, None) == _lib.PA_EINVAL
        assert b"null" in lib.pa_last_error()


def test_rfft_f32_overlap_is_sized_with_4_and_8_byte_elements():
    """16 x 6 x 4 Float32 = 1536 bytes, 9 x 6 x 4 ComplexF32 = 1728 bytes: overlaps by one
    element are refused, adjacent arrays are not -- at the single-precision sizes, which the
    double-precision sizes (twice as large) would get wrong."""
    pr, pc = _pencils()
    rb, cb = _bytes(pr, pc)
    assert (rb, cb) == (16 * 24 * 4, 9 * 24 * 8)
    buf = HostBuf(4 * (rb + cb))
    for flags, nsrc, ndst in ((FWD, rb, cb), (BWD, cb, rb)):
        for s, d in ((0, nsrc - 16), (ndst - 16, 0), (0, 0)):
            assert lib.pa_rfft(pr._h, pc._h, 0, None, flags | F32, buf.at(s), buf.at(d), None) \
                == _lib.PA_EINVAL, (flags, s, d)
            assert b"overlap" in lib.pa_last_error()
        # adjacent: past the overlap check (rb and cb are multiples of 16)
        st = lib.pa_rfft(pr._h, pc._h, 0, None, flags | F32, buf.at(0), buf.at(nsrc), None)
        assert st != _lib.PA_EINVAL or b"overlap" not in lib.pa_last_error()
        if no_gpu():
            assert st == _lib.PA_ENOGPU
            # dst right behind src at the double-precision size would overlap; at fp32 it is free
            assert lib.pa_rfft(pr._h, pc._h, 0, None, flags | F32, buf.at(ndst), buf.at(0), None) \
                == _lib.PA_ENOGPU
        # misaligned by 8 (or 4) bytes
        for s, d in ((8, nsrc + 16), (0, nsrc + 8), (4, nsrc + 16)):
            assert lib.pa_rfft(pr._h, pc._h, 0, None, flags | F32, buf.at(s), buf.at(d), None) \
                == _lib.PA_EINVAL
            assert b"aligned" in lib.pa_last_error()


def test_rfft_f32_extra_dims_limits():
    pr, pc = _pencils()
    buf = HostBuf(1 << 16)
    assert lib.pa_rfft(pr._h, pc._h, 6, i64arr((1, 1, 1, 1, 1, 2)), FWD | F32, buf.at(0),
                       buf.at(1 << 15), None) == _lib.PA_EINVAL
    assert lib.pa_rfft(pr._h, pc._h, 1, i64arr((-2,)), FWD | F32, buf.at(0), buf.at(1 << 15),
                       None) == _lib.PA_EINVAL


# ---- Python wrappers (CPU tensors stand in for the parent arrays) ---------------------------
def _arr(p, dtype, *extra):
    mem = pa.size_local(p, pa.MemoryOrder())
    return pa.PencilArray(p, torch.zeros(tuple(reversed(mem + extra)), dtype=dtype), extra)


def test_python_rfft_accepts_the_single_precision_pair():
    """(float32, complex64) passes the wrapper's dtype check and goes on to the device (which
    this CPU-only run lacks: the error is not an ArgumentError); the mixed pairs stay refused."""
    if not no_gpu():
        pytest.skip("GPU present: CPU tensors must not reach the library")
    pr, pc = _pencils()
    xr, xc = _arr(pr, torch.float32), _arr(pc, torch.complex64)
    for call in (lambda: pa.rfft_(xc, xr), lambda: pa.brfft_(xr, xc)):
        with pytest.raises(Exception) as e:
            call()
        assert not isinstance(e.value, pa.ArgumentError), e.value
    for bad in (lambda: pa.rfft_(_arr(pc, torch.complex128), xr),
                lambda: pa.rfft_(xc, _arr(pr, torch.float64)),
                lambda: pa.brfft_(_arr(pr, torch.float64), xc),
                lambda: pa.brfft_(xr, _arr(pc, torch.complex128))):
        with pytest.raises(pa.ArgumentError):
            bad()


def test_python_fft_fusable_follows_the_dtype():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    px = pa.Pencil(topo, (16, 8, 4), (2, 3))
    py = pa.Pencil(px, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    for dtype, ok in ((torch.complex64, True), (torch.complex128, True), (torch.float64, False),
                      (torch.float32, False)):
        t = pa.Transposition(_arr(py, dtype), _arr(px, dtype))
        assert t.fft_fusable() is ok, dtype
    # 12-point lines: refused in either precision
    qx = pa.Pencil(topo, (16, 12, 4), (2, 3))
    qy = pa.Pencil(qx, decomp_dims=(1, 3), permute=pa.Permutation(2, 1, 3))
    for dtype in (torch.complex64, torch.complex128):
        assert not pa.Transposition(_arr(qy, dtype), _arr(qx, dtype)).fft_fusable()
