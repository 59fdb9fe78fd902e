"""Global reductions on the GPU (pa_reduce, reductions.py), one process:

* every element type x map x op against numpy on a permuted pencil of odd sizes (16, 21, 41) with
  extra dims, on a view one element off the allocation's alignment, and n from 0 to 256 MiB:
  integers, max, min, any and all exact (abs of complex values within one ulp of numpy's hypot),
  float sums within depth eps sum|f(x)| of math.fsum, depth the tree depth reduce.cu documents;
* two calls bitwise equal, exactly one launch per call;
* a refused call launches nothing and leaves a guard-banded result buffer untouched;
* stream ordering without host synchronisation (the gpu_util.hold() pattern);
* tests/mp_reduce_worker.py with 2, 3, 4 and 8 processes sharing the GPU, and the NCCL fallback
  where two GPUs exist."""
import ctypes as C
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

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DIMS = (16, 21, 41)
TYPES = [torch.float64, torch.float32, torch.complex128, torch.complex64, torch.int32, torch.int64]


def depth(n, elsize, P=1):
    """The Float64 sum's tree depth of reduce.cu's header for n elements on this device."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nunits = n * elsize // 16
    G = max(1, min(math.ceil(n * elsize / 16 / 1024), 4 * sms))
    run = math.ceil(math.ceil(nunits / G) / 256) * (16 // elsize) + 2
    return run + 5 + 3 + math.ceil(G / 256) + 5 + 3 + (P - 1)


def make(dtype, pen, extra=(), offset=0, seed=0):
    """A PencilArray whose data starts `offset` elements into its allocation, and its numpy copy."""
    rng = np.random.default_rng(seed)
    mem = pa.size_local(pen, pa.MemoryOrder())
    shape = tuple(reversed(mem + tuple(extra)))
    n = math.prod(shape)
    if dtype.is_complex:
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    elif dtype.is_floating_point:
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 3, n)
    else:
        x = rng.integers(-60000, 60000, n)
    x = x.astype(torch.empty(0, dtype=dtype).numpy().dtype)
    buf = torch.empty(n + offset, dtype=dtype, device="cuda")
    buf[offset:].copy_(torch.from_numpy(x))
    return pa.PencilArray(pen, buf[offset:].view(shape), tuple(extra)), x


def mapped(x, f):
    if f is None:
        return x
    if f is abs:
        return np.abs(x)
    if np.iscomplexobj(x):
        return x.real * x.real + x.imag * x.imag
    with np.errstate(over="ignore"):
        return x * x  # integers wrap, as Julia's abs2


def check_one(u, x, f, op):
    got = {"+": pa.sum, "max": pa.maximum, "min": pa.minimum}[op](u, f)
    assert got.dim() == 0 and got.device == u.data.device
    fx = mapped(x, f)
    if op != "+":
        want = fx.max() if op == "max" else fx.min()
        if f is abs and np.iscomplexobj(x):
            assert abs(got.item() - want) <= np.spacing(want), (f, op)
        else:
            assert got.item() == want, (f, op)
        return
    if not got.dtype.is_floating_point and not got.dtype.is_complex:
        assert got.dtype == torch.int64
        assert got.item() == int(fx.astype(np.int64).sum()), (f, op)
        return
    for part, g in ((lambda a: a.real, got.real if got.is_complex() else got),
                    (lambda a: a.imag, got.imag if got.is_complex() else None)):
        if g is None:
            continue
        fp = part(fx).astype(np.float64)
        want = math.fsum(fp)
        tol = depth(len(x), x.itemsize) * np.finfo(np.float64).eps * math.fsum(np.abs(fp))
        if g.dtype == torch.float32:
            tol += float(np.spacing(np.float32(abs(want))))
        assert abs(g.item() - want) <= tol, (f, op, g.item(), want, tol)


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("offset", [0, 1])
def test_every_map_and_op_against_numpy(dtype, offset):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, DIMS, (2, 3), permute=pa.Permutation(3, 1, 2))
    for extra in ((), (3,), (2, 2)):
        u, x = make(dtype, pen, extra, offset, seed=len(extra))
        for f in (None, abs, pa.abs2):
            for op in ("+", "max", "min"):
                if dtype.is_complex and f is None and op != "+":
                    with pytest.raises(pa.ArgumentError, match="not ordered"):
                        pa.mapreduce(f, op, u)
                    continue
                check_one(u, x, f, op)
        d = pa.mapreduce(pa.realdot, "+", u, u)
        assert d.cpu().numpy().tobytes() == pa.sum(u, pa.abs2).cpu().numpy().tobytes()
        v, y = make(dtype, pen, extra, 0, seed=9)
        got = pa.mapreduce(pa.realdot, "+", u, v)
        prod = (x * np.conj(y)).real if dtype.is_complex else x.astype(np.float64) * y
        if got.dtype == torch.int64:
            assert got.item() == int((x.astype(np.int64) * y.astype(np.int64)).astype(
                x.dtype).astype(np.int64).sum())
        else:
            tol = depth(len(x), x.itemsize) * np.finfo(np.float64).eps * math.fsum(np.abs(prod)) * 4
            if got.dtype == torch.float32:
                tol += 64 * float(np.finfo(np.float32).eps) * math.fsum(np.abs(prod))
            assert abs(got.item() - math.fsum(prod)) <= tol
        # any / all, exact
        v0 = x.flat[17]
        assert pa.any(u, "==", v0).item() is True
        assert pa.all(u, "!=", v0).item() is False
        assert pa.all(u, "isfinite").item() is True and pa.any(u, "isnan").item() is False
        if not dtype.is_complex:
            assert pa.all(u, ">=", x.min()).item() is True
            assert pa.all(u, ">", x.min()).item() is False
            assert pa.any(u, "<", x.min()).item() is False
            assert pa.any(u, "<=", x.min()).item() is True
        bound = np.abs(x).max() if not dtype.is_floating_point and not dtype.is_complex else \
            np.abs(x).max() * np.abs(x).dtype.type(1.0001)  # (a value of the mapped type)
        assert pa.all(u, "<=", bound, f=abs).item() is True


@pytest.mark.parametrize("n", [0, 1, 3, 1023, 4097, 1 << 20, (256 << 20) // 8])
def test_sizes(n):
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, (n, 1, 1), (2, 3))
    u, x = make(torch.float64, pen, (), 0, seed=n)
    if n == 0:
        assert pa.sum(u).item() == 0.0
    assert pa.any(u, "isnan").item() is False and pa.all(u, "isfinite").item() is True
    if n == 0:
        for fn in (pa.maximum, pa.minimum):
            with pytest.raises(pa.ArgumentError, match="empty collection"):
                fn(u)
        return
    for f in (None, abs, pa.abs2):
        check_one(u, x, f, "+")
    check_one(u, x, abs, "max")
    check_one(u, x, None, "min")


def test_float32_threshold_compares_in_the_element_type():
    """Values Float32 holds exactly compare as Julia does; others are refused (0.1 is not
    0.1f0: Julia's any(>(0.1), u) compares in Float64)."""
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, (100, 3, 1), (2, 3))
    u = pa.PencilArray.undef(torch.float32, pen)
    u.data.fill_(0.1)
    assert pa.any(u, "==", np.float32(0.1)).item() is True
    assert pa.any(u, ">", 0.09375).item() is True and pa.all(u, "<", 0.125).item() is True
    with pytest.raises(pa.ArgumentError, match="not exactly representable"):
        pa.any(u, ">", 0.1)


def test_nan_and_signed_zero():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, (1000, 3, 1), (2, 3))
    u, x = make(torch.float64, pen)
    u.data.view(-1)[1777] = float("nan")
    assert math.isnan(pa.maximum(u).item()) and math.isnan(pa.minimum(u).item())
    assert pa.any(u, "isnan").item() is True and pa.all(u, "isfinite").item() is False
    u.data.fill_(-0.0)
    u.data.view(-1)[2001] = 0.0
    assert math.copysign(1, pa.maximum(u).item()) == 1.0
    assert math.copysign(1, pa.minimum(u).item()) == -1.0


@pytest.mark.parametrize("ctype", [torch.complex128, torch.complex64])
def test_complex_arrays_off_their_element_alignment_through_the_c_abi(ctype):
    """ComplexF64 at an odd 8 bytes and ComplexF32 at an odd 4 bytes (aligned to their real
    component only): every element is loaded alone.  Every map and op on that path, the second
    array of realdot at the same and at another alignment."""
    rt = torch.float64 if ctype == torch.complex128 else torch.float32
    npc = np.complex128 if ctype == torch.complex128 else np.complex64
    dt = _lib.PA_COMPLEXF64 if ctype == torch.complex128 else _lib.PA_COMPLEXF32
    comp = torch.empty(0, dtype=rt).element_size()
    n = 4097
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, (n, 1, 1), (2, 3))
    raw = torch.randn(2 * (2 * n + 1), dtype=rt, device="cuda")
    a_ptr = raw.data_ptr() + comp                        # odd component: not element-aligned
    b_other = raw.data_ptr() + (2 * n + 2) * comp        # element-aligned: another alignment
    hb = raw.cpu().numpy()
    x = hb[1:2 * n + 1].view(npc)
    y = hb[2 * n + 2:4 * n + 2].view(npc)
    x0 = x[17].copy()

    def call(f, op, result, pred=None, b=None):
        st = lib.pa_reduce(pen._h, 0, None, None, dt, f, op,
                           None if pred is None else C.c_void_p(pred.data_ptr()), C.c_void_p(a_ptr),
                           None if b is None else C.c_void_p(b), C.c_void_p(result.data_ptr()),
                           stream_ptr())
        assert st == 0, lib.pa_last_error().decode()
        torch.cuda.synchronize()
        return result.item()

    eps = float(np.finfo(np.float64).eps)
    tolr = depth(n, 2 * comp) * eps + (float(np.finfo(np.float32).eps) if comp == 4 else 0)
    r_c = torch.empty((), dtype=ctype, device="cuda")
    r_r = torch.empty((), dtype=rt, device="cuda")
    r_b = torch.empty((), dtype=torch.bool, device="cuda")
    s = call(_lib.PA_MAP_IDENTITY, _lib.PA_OP_SUM, r_c)
    xd = x.astype(np.complex128)
    for got, want, mag in ((s.real, math.fsum(xd.real), math.fsum(abs(xd.real))),
                           (s.imag, math.fsum(xd.imag), math.fsum(abs(xd.imag)))):
        assert abs(got - want) <= tolr * mag
    ab, a2 = np.abs(x), x.real * x.real + x.imag * x.imag
    for f, v in ((_lib.PA_MAP_ABS, ab), (_lib.PA_MAP_ABS2, a2)):
        vd = v.astype(np.float64)
        assert abs(call(f, _lib.PA_OP_SUM, r_r) - math.fsum(vd)) <= tolr * math.fsum(vd)
        for op, want in ((_lib.PA_OP_MAX, v.max()), (_lib.PA_OP_MIN, v.min())):
            got = call(f, op, r_r)
            if f == _lib.PA_MAP_ABS:
                assert abs(got - want) <= np.spacing(want)
            else:
                assert got == want
    pv = torch.tensor([complex(x0)], dtype=ctype)
    assert call(_lib.PA_MAP_IDENTITY, _lib.PA_OP_ANY | _lib.PA_PRED_EQ, r_b, pv) is True
    assert call(_lib.PA_MAP_IDENTITY, _lib.PA_OP_ALL | _lib.PA_PRED_NE, r_b, pv) is False
    assert call(_lib.PA_MAP_IDENTITY, _lib.PA_OP_ANY | _lib.PA_PRED_ISNAN, r_b) is False
    assert call(_lib.PA_MAP_IDENTITY, _lib.PA_OP_ALL | _lib.PA_PRED_ISFINITE, r_b) is True
    # realdot(x, x) is abs2 bit for bit; with y at another alignment against numpy
    r_s = torch.empty((), dtype=rt, device="cuda")
    call(_lib.PA_MAP_ABS2, _lib.PA_OP_SUM, r_s)
    call(_lib.PA_MAP_DOT, _lib.PA_OP_SUM, r_r, b=a_ptr)
    assert r_r.cpu().numpy().tobytes() == r_s.cpu().numpy().tobytes()
    prod = (xd * np.conj(y.astype(np.complex128))).real
    got = call(_lib.PA_MAP_DOT, _lib.PA_OP_SUM, r_r, b=b_other)
    assert abs(got - math.fsum(prod)) <= (4 * tolr + (64e-7 if comp == 4 else 0)) * math.fsum(abs(prod))


def test_two_calls_bitwise_equal_and_one_launch_each():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, (512, 256, 33), (2, 3))
    for dtype in (torch.float64, torch.complex64):
        u, _ = make(dtype, pen, (2,))
        a = pa.sum(u)
        n0 = pa.launch_count()
        b = pa.sum(u)
        assert pa.launch_count() - n0 == 1
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
        n0 = pa.launch_count()
        pa.maximum(u, abs)
        pa.all(u, "isfinite")
        assert pa.launch_count() - n0 == 2


def test_refused_call_launches_nothing_and_leaves_the_result_untouched():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, DIMS, (2, 3))
    u, _ = make(torch.complex128, pen)
    guard = torch.full((48,), 0x5A, dtype=torch.uint8, device="cuda")
    res = C.c_void_p(guard.data_ptr() + 16)
    n0 = pa.launch_count()
    cases = [
        (_lib.PA_COMPLEXF64, _lib.PA_MAP_IDENTITY, _lib.PA_OP_MAX, None, None),   # not ordered
        (_lib.PA_COMPLEXF64, _lib.PA_MAP_DOT, _lib.PA_OP_SUM, None, None),        # b missing
        (_lib.PA_COMPLEXF64, _lib.PA_MAP_ABS, _lib.PA_OP_ANY | _lib.PA_PRED_GT, None, None),
    ]
    for dt, f, op, pred, b in cases:
        assert lib.pa_reduce(pen._h, 0, None, None, dt, f, op, pred, C.c_void_p(u.data_ptr()), b,
                             res, stream_ptr()) == _lib.PA_EINVAL
    h = C.c_void_p()
    assert lib.pa_comm_init_local(2, 0, C.byref(h)) == 0
    try:
        assert lib.pa_reduce(pen._h, 0, None, h, _lib.PA_COMPLEXF64, _lib.PA_MAP_ABS, _lib.PA_OP_SUM,
                             None, C.c_void_p(u.data_ptr()), None, res,
                             stream_ptr()) == _lib.PA_EINCOMPAT
        assert "the communicator 2" in lib.pa_last_error().decode()
    finally:
        lib.pa_comm_destroy(h)
    assert pa.launch_count() == n0
    torch.cuda.synchronize()
    assert bool((guard == 0x5A).all())


def test_stream_ordering_without_host_sync():
    topo = pa.MPITopology(pa.COMM_SELF, (1, 1))
    pen = pa.Pencil(topo, (256, 128, 64), (2, 3))
    u = pa.PencilArray.undef(torch.float64, pen)
    u.data.fill_(1.0)
    pa.sum(u)  # warm-up
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        held = hold()
        u.data.fill_(2.0)          # produced behind the hold
        r = pa.sum(u)
        m = pa.maximum(u)
        assert not held.query()    # the calls did not wait for the device
    torch.cuda.synchronize()
    assert r.item() == 2.0 * u.data.numel() and m.item() == 2.0


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
# the same kernel once through a one-rank communicator (which has a workspace of its own), so that
# what follows measures the device workspace's setup alone
h = C.c_void_p()
assert lib.pa_comm_init_local(1, 0, C.byref(h)) == 0
res = torch.empty((), dtype=torch.float64, device="cuda")
assert lib.pa_reduce(pen._h, 0, None, h, 0, 0, 0, None, C.c_void_p(u.data_ptr()), None,
                     C.c_void_p(res.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
torch.cuda.synchronize()
held = hold()
u.data.fill_(1.0)
r = pa.sum(u)  # the first reduction on this device: it sets up its workspace
assert not held.query(), "the first reduction synchronised the host"
assert r.item() == 64 * 32 * 16
print("FIRST_CALL_OK")
'''


def test_first_one_rank_call_does_not_synchronise_the_host():
    """In a fresh process, so that the device's workspace does not exist yet."""
    out = subprocess.run([sys.executable, "-c", FIRST_CALL, os.path.dirname(HERE), HERE],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "FIRST_CALL_OK" in out.stdout, out.stderr[-2000:]


def _run_workers(nproc, tmp_path, env_extra=None, port=29751):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port + nproc),
           os.path.join(HERE, "mp_reduce_worker.py")]
    env = dict(os.environ, OMP_NUM_THREADS="1", **(env_extra or {}))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    errs = [l for l in out.stderr.splitlines() if l.startswith("WORKER-ERROR")]
    assert out.returncode == 0, "\n".join(errs[-60:]) + out.stdout[-1500:] + out.stderr[-1500:]
    return out.stdout


@pytest.mark.parametrize("nproc", [2, 3, 4, 8])
def test_ranks_sharing_the_gpu(nproc, tmp_path):
    out = _run_workers(nproc, tmp_path)
    assert f"MP_REDUCE_OK world={nproc} nccl=0" in out, out[-2000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="the NCCL fallback needs >= 2 GPUs")
def test_nccl_fallback(tmp_path):
    out = _run_workers(2, tmp_path, {"PA_REDUCE_NCCL": "1", "PA_B200_TRANSPORT": "nccl"}, port=29771)
    assert "MP_REDUCE_OK world=2 nccl=1" in out, out[-2000:]
