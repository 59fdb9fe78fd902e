"""Reductions along dims on the GPU (pa_reduce_dims, the ``dims`` keyword of reductions.py), one
process, against numpy on ``u.logical()`` (tests/reduce_dims_ref.py):

* pencils with the permutations identity, (2, 1, 3) and (3, 2, 1) and 0 to 2 extra dims, every
  non-empty subset of dims, all six element types, every map / op / predicate;
* odd and extent-1 sizes, empty local arrays, bases off the 16-byte alignment;
* few outputs with many inputs (keep a dim of 3 over 512 x 512) and many outputs with few inputs;
* integers, max / min and any / all exact (NaN and -0.0 included), float sums within the bound of
  DESIGN §3l against math.fsum per element;
* two calls bitwise equal, one launch each; a refused call launches nothing and leaves the result
  untouched; stream ordering without host synchronisation, also for the first call in a process;
* dims covering every dim equal pa_reduce bit for bit;
* tests/mp_reduce_dims_worker.py with 2, 3, 4 and 8 processes sharing the GPU."""
import ctypes as C
import itertools
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib
from gpu_util import hold, stream_ptr
from reduce_dims_ref import expect, check, logical_view

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TYPES = [torch.float64, torch.float32, torch.complex128, torch.complex64, torch.int32, torch.int64]
SELF = (1, 1)


def pencil(dims, perm=None):
    kw = {"permute": pa.Permutation(*perm)} if perm else {}
    return pa.Pencil(pa.MPITopology(pa.COMM_SELF, SELF), dims, (2, 3), **kw)


def make(dtype, pen, extra=(), offset=0, seed=0, special=False):
    """A PencilArray `offset` elements into its allocation, and its logical-order numpy copy."""
    rng = np.random.default_rng(seed)
    mem = pa.size_local(pen, pa.MemoryOrder())
    shape = tuple(reversed(mem + tuple(extra)))
    n = math.prod(shape)
    if dtype.is_complex:
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    elif dtype.is_floating_point:
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 3, n)
        if special and n:
            k = rng.integers(0, n, max(1, n // 7))
            x[k] = rng.choice([0.0, -0.0, np.nan, np.inf, -np.inf], len(k))
    else:
        x = rng.integers(-60000, 60000, n)
    x = x.astype(torch.empty(0, dtype=dtype).numpy().dtype)
    buf = torch.empty(n + offset, dtype=dtype, device="cuda")
    buf[offset:].copy_(torch.from_numpy(x))
    u = pa.PencilArray(pen, buf[offset:].view(shape), tuple(extra))
    return u, logical_view(u, u.data).cpu().numpy()


def cases(dtype):
    """(f, op, pred, value) of every map / op / predicate the element type allows."""
    cplx = dtype.is_complex
    out = [(f, "+", None, None) for f in (None, abs, pa.abs2)]
    out += [(f, op, None, None) for f in ((abs, pa.abs2) if cplx else (None, abs, pa.abs2))
            for op in ("max", "min")]
    preds = [("==", 0), ("!=", 0), ("isnan", None), ("isfinite", None)]
    if not cplx:
        preds += [("<", 0), ("<=", 0), (">", 0), (">=", 0)]
    out += [(None, op, p, v) for op in ("any", "all") for p, v in preds]
    out += [(abs, "any", ">", 1)]
    return out


def run(u, f, op, dims, pred=None, value=None):
    if op in ("any", "all"):
        return getattr(pa, op)(u, pred, value, f=f, dims=dims)
    return {"+": pa.sum, "max": pa.maximum, "min": pa.minimum}[op](u, f, dims=dims)


def check_all(u, x, dims, what, only=None):
    for f, op, pred, value in (only or cases(u.dtype)):
        got = run(u, f, op, dims, pred, value)
        # the dtype the mirror allocated is the library's result type
        assert got.dtype == (torch.bool if op in ("any", "all") else
                             pa.reductions.result_dtype(u.dtype, f, op)), (f, op)
        want, tol = expect(x, f, op, dims, pred, value)
        if f is abs and u.dtype.is_complex and op in ("max", "min"):
            tol = 2 * np.abs(np.spacing(want))  # hypot within an ulp of numpy's (either candidate)
        check(logical_view(u, got).cpu().numpy(), want, tol, (what, f, op, pred, dims))


def subsets(n):
    return [s for k in range(1, n + 1) for s in itertools.combinations(range(1, n + 1), k)]


@pytest.mark.parametrize("perm,extra", [(None, ()), ((2, 1, 3), (2,)), ((3, 2, 1), (3, 2)),
                                        (None, (1, 2)), ((2, 3, 1), (2,)), ((3, 1, 2), ())])
@pytest.mark.parametrize("dtype", TYPES)
def test_every_subset_map_and_op_against_numpy(perm, extra, dtype):
    pen = pencil((7, 5, 6), perm)
    u, x = make(dtype, pen, extra, seed=len(extra))
    for dims in subsets(3 + len(extra)):
        check_all(u, x, dims, (perm, extra))


@pytest.mark.parametrize("boff", [0, 1, 2])
@pytest.mark.parametrize("dtype", TYPES)
def test_realdot_every_subset(dtype, boff):
    """mapreduce(realdot, +, u, v; dims): `v` at the same 16-byte alignment as `u` (16-byte units
    on both arrays) and at another one (element loads); a 3-cycle permutation and an extra dim;
    row-regime rows of 64 and 5 elements."""
    for size, perm in (((64, 5, 6), (2, 3, 1)), ((64, 3, 7), None)):
        pen = pencil(size, perm)
        u, x = make(dtype, pen, (2,), seed=1)
        v, y = make(dtype, pen, (2,), offset=boff, seed=2)
        for dims in subsets(4):
            got = pa.mapreduce(pa.realdot, "+", u, v, dims=dims)
            assert got.dtype == pa.reductions.result_dtype(dtype, pa.realdot, "+")
            want, tol = expect(x, pa.realdot, "+", dims, y=y)
            check(logical_view(u, got).cpu().numpy(), want, tol, (size, perm, boff, dims))
        # realdot of u with itself is sum(abs2) bit for bit
        for dims in ((1,), (2, 3), (4,)):
            a = pa.mapreduce(pa.realdot, "+", u, u, dims=dims)
            b = pa.sum(u, pa.abs2, dims=dims)
            assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


@pytest.mark.parametrize("dtype", TYPES)
def test_offset_bases_and_odd_sizes(dtype):
    for off, size, perm in ((1, (33, 9, 5), None), (3, (64, 3, 17), (2, 1, 3)),
                            (1, (1, 40, 3), (3, 2, 1))):
        pen = pencil(size, perm)
        u, x = make(dtype, pen, (2,), offset=off, seed=off)
        for dims in ((1,), (2,), (1, 3), (2, 3, 4), (1, 4)):
            check_all(u, x, dims, (off, size), only=cases(dtype)[:4])


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_nan_and_signed_zero(dtype):
    pen = pencil((40, 9, 7), (2, 1, 3))
    u, x = make(dtype, pen, (2,), special=True, seed=5)
    for dims in subsets(4):
        check_all(u, x, dims, "special", only=[(None, "max", None, None), (None, "min", None, None),
                                               (None, "any", "isnan", None),
                                               (None, "all", "isfinite", None),
                                               (None, "any", "==", 0)])


@pytest.mark.parametrize("dtype", [torch.float64, torch.complex128, torch.float32, torch.int32])
def test_extremes(dtype):
    """Few outputs with many inputs (each output split over CTAs), many outputs with few inputs."""
    for size, perm, dims in (((3, 512, 512), None, (2, 3)),      # keep x: the column regime
                             ((512, 3, 512), None, (1, 3)),      # keep y
                             ((512, 512, 3), None, (1, 2)),      # keep z: one long row
                             ((2, 300, 301), None, (1,)),        # reduce 2 contiguous
                             ((300, 2, 301), (2, 1, 3), (1,))):  # reduce 2 strided
        pen = pencil(size, perm)
        u, x = make(dtype, pen, seed=7)
        check_all(u, x, dims, size, only=[(None, "+", None, None), (abs, "max", None, None),
                                          (None, "any", "isfinite", None)])


def test_empty_local_arrays_and_results():
    pen = pencil((0, 5, 4))
    u, x = make(torch.float64, pen)
    r = pa.sum(u, dims=(1,))          # a sum over an empty range: zeros
    assert r.shape == (4, 5, 1) and bool((r == 0).all())
    r = pa.sum(u, dims=(2, 3))        # an empty result
    assert r.shape == (1, 1, 0)
    r = pa.maximum(u, dims=(2,))      # empty result: allowed
    assert r.numel() == 0
    with pytest.raises(pa.ArgumentError, match="empty collection"):
        pa.maximum(u, dims=(1,))
    torch.cuda.synchronize()


def test_every_dim_is_pa_reduce():
    pen = pencil((17, 9, 13), (3, 2, 1))
    for dtype in TYPES:
        u, _ = make(dtype, pen, (2,), offset=1)
        for f, op, pred, value in cases(dtype):
            a = run(u, f, op, None, pred, value)
            b = run(u, f, op, (4, 2, 3, 1), pred, value)
            assert b.shape == (1, 1, 1, 1)
            assert a.reshape(1).cpu().numpy().tobytes() == b.reshape(1).cpu().numpy().tobytes()


def test_two_calls_bitwise_equal_and_one_launch_each():
    pen = pencil((512, 256, 33))
    for dtype in (torch.float64, torch.complex64):
        u, _ = make(dtype, pen, (2,))
        for dims in ((1,), (2, 3), (3,), (1, 4)):
            a = pa.sum(u, dims=dims)
            n0 = pa.launch_count()
            b = pa.sum(u, dims=dims)
            assert pa.launch_count() - n0 == 1
            assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
            n0 = pa.launch_count()
            pa.maximum(u, abs, dims=dims)
            pa.all(u, "isfinite", dims=dims)
            assert pa.launch_count() - n0 == 2


def test_refused_call_launches_nothing_and_leaves_the_result_untouched():
    pen = pencil((16, 21, 41))
    u, _ = make(torch.float64, pen)
    guard = torch.full((16 * 21 * 8 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    res = C.c_void_p(guard.data_ptr() + 32)
    n0 = pa.launch_count()

    def call(dims, op=_lib.PA_OP_SUM, comm=None):
        arr = (C.c_int * max(1, len(dims)))(*dims)
        return lib.pa_reduce_dims(pen._h, 0, None, comm, _lib.PA_FLOAT64, _lib.PA_MAP_IDENTITY, op,
                                  None, C.c_void_p(u.data_ptr()), None, len(dims), arr, res,
                                  stream_ptr())
    for dims in ((), (0,), (4,), (1, 1), (2, -1)):
        assert call(dims) == _lib.PA_EINVAL, dims
    h = C.c_void_p()
    assert lib.pa_comm_init_local(2, 0, C.byref(h)) == 0
    try:
        assert call((3,), comm=h) == _lib.PA_EINCOMPAT
    finally:
        lib.pa_comm_destroy(h)
    assert pa.launch_count() == n0
    torch.cuda.synchronize()
    assert bool((guard == 0x5A).all())


def test_stream_ordering_without_host_sync():
    pen = pencil((256, 128, 64))
    u = pa.PencilArray.undef(torch.float64, pen)
    u.data.fill_(1.0)
    pa.sum(u, dims=(1,))  # warm-up
    pa.sum(u, dims=(2,))
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        held = hold()
        u.data.fill_(2.0)          # produced behind the hold
        r = pa.sum(u, dims=(1,))
        m = pa.maximum(u, dims=(2,))
        assert not held.query()    # the calls did not wait for the device
    torch.cuda.synchronize()
    assert bool((r == 512.0).all()) and bool((m == 2.0).all())


FIRST_CALL = r'''
import sys, torch
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import pencilarrays_b200 as pa
from gpu_util import hold, hold_cycles
import ctypes as C
from pencilarrays_b200._lib import lib
hold_cycles()
pen = pa.Pencil(pa.MPITopology(pa.COMM_SELF, (1, 1)), (64, 32, 16), (2, 3))
u = pa.PencilArray.undef(torch.float64, pen)
u.data.fill_(0.0)
# CUDA loads a kernel's module at its first launch, and that load waits for the device: launch
# the same kernel once through a one-rank communicator (which has a workspace of its own)
h = C.c_void_p()
assert lib.pa_comm_init_local(1, 0, C.byref(h)) == 0
res = torch.empty((16, 1, 64), dtype=torch.float64, device="cuda")
dims = (C.c_int * 1)(2)
assert lib.pa_reduce_dims(pen._h, 0, None, h, 0, 0, 0, None, C.c_void_p(u.data_ptr()), None, 1,
                          dims, C.c_void_p(res.data_ptr()),
                          C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
torch.cuda.synchronize()
held = hold()
u.data.fill_(1.0)
r = pa.sum(u, dims=2)  # the first reduction on this device: it sets up its workspace
assert not held.query(), "the first reduction synchronised the host"
assert bool((r == 32).all()) and r.shape == (16, 1, 64)
print("FIRST_CALL_OK")
'''


def test_first_one_rank_call_does_not_synchronise_the_host():
    """In a fresh process, so that the device's workspace does not exist yet."""
    out = subprocess.run([sys.executable, "-c", FIRST_CALL, os.path.dirname(HERE), HERE],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "FIRST_CALL_OK" in out.stdout, out.stderr[-2000:]


@pytest.mark.parametrize("nproc", [2, 3, 4, 8])
def test_ranks_sharing_the_gpu(nproc):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29811 + nproc),
           os.path.join(HERE, "mp_reduce_dims_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    assert f"MP_REDUCE_DIMS_OK world={nproc}" in out.stdout, out.stdout[-2000:]
