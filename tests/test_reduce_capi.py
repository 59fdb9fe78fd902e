"""pa_reduce / pa_reduce_result_type on the host (no GPU needed): the whole result-type table,
every refusal with its pa_last_error text, PA_ENOGPU for a valid call on a machine without a GPU
(on one with a GPU a valid call would run, so those cases are checked only there), and the
Python mirror's ArgumentError for incompatible arrays."""
import ctypes as C
import itertools
import math

import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, i64arr

F64, F32, C64, C32, I32, I64, BOOL = range(7)
ID, ABS, ABS2, DOT = range(4)
SUM, MAX, MIN, ANY, ALL = range(5)
EQ, NE, LT, LE, GT, GE, ISNAN, ISFINITE = (k << 4 for k in range(1, 9))
PREDS = (EQ, NE, LT, LE, GT, GE, ISNAN, ISFINITE)
REAL = {C64: F64, C32: F32}
NO_GPU = lib.pa_device_count() == 0


def expected(dtype, f, op):
    """Julia's table: None where the combination is refused."""
    base, p = op & 15, op >> 4
    cval = dtype in (C64, C32) and f == ID
    val = dtype if cval else REAL.get(dtype, dtype)
    if base in (ANY, ALL):
        if p == 0 or (cval and (LT >> 4) <= p <= (GE >> 4)):
            return None
        return BOOL
    if p != 0 or (cval and base in (MAX, MIN)):
        return None
    return I64 if base == SUM and val == I32 else val


def result_type(dtype, f, op):
    out = C.c_int(-1)
    s = lib.pa_reduce_result_type(dtype, f, op, C.byref(out))
    return s, out.value


def test_result_type_table():
    ops = [SUM, MAX, MIN] + [b | p for b in (ANY, ALL) for p in PREDS] + [ANY, ALL, SUM | EQ]
    for dtype, f, op in itertools.product(range(6), range(4), ops):
        want = expected(dtype, f, op)
        s, got = result_type(dtype, f, op)
        if want is None:
            assert s == _lib.PA_EINVAL, (dtype, f, op)
            assert lib.pa_last_error().decode().startswith("pa_reduce:")
        else:
            assert (s, got) == (_lib.PA_OK, want), (dtype, f, op)
    for bad in ((7, ID, SUM), (-1, ID, SUM), (F64, 4, SUM), (F64, ID, 5), (F64, ID, ANY | (9 << 4))):
        assert result_type(*bad)[0] == _lib.PA_EINVAL, bad
    assert "not ordered" in (lib.pa_reduce_result_type(C64, ID, MAX, None) and
                             lib.pa_last_error().decode())


def test_python_result_dtype_asks_the_library():
    assert pa.reductions.result_dtype(torch.int32) == torch.int64
    assert pa.reductions.result_dtype(torch.complex64, abs) == torch.float32
    assert pa.reductions.result_dtype(torch.complex128, pa.abs2) == torch.float64
    assert pa.reductions.result_dtype(torch.float32, None, max) == torch.float32
    with pytest.raises(pa.ArgumentError, match="not ordered"):
        pa.reductions.result_dtype(torch.complex128, None, max)


@pytest.fixture(scope="module")
def pens():
    one = pa.Pencil(pa.MPITopology(pa.COMM_SELF, (1, 1)), (16, 21, 41), (2, 3))
    empty = pa.Pencil(pa.MPITopology(pa.COMM_SELF, (1, 1)), (16, 0, 41), (2, 3))
    four = pa.Pencil(pa.MPITopology(pa.Comm(0, 4), (2, 2)), (16, 21, 41), (2, 3))
    return one, empty, four


A = C.c_void_p(0x10000)   # stand-ins: these checks never touch the memory
B = C.c_void_p(0x20000)
R = C.c_void_p(0x30000)
VAL = C.c_double(1.0)


def call(pen, dtype=F64, f=ID, op=SUM, a=A, b=None, result=R, pred=None, n_extra=0, extra=(),
         comm=None):
    return lib.pa_reduce(pen._h, n_extra, i64arr(extra), comm, dtype, f, op,
                         C.byref(pred) if pred is not None else None, a, b, result, None)


def refused(status, text, *args, **kw):
    s = call(*args, **kw)
    err = lib.pa_last_error().decode()
    assert s == status and text in err, (s, err)


def test_refusals(pens):
    one, empty, four = pens
    n0 = lib.pa_launch_count()
    refused(_lib.PA_EINVAL, "null pencil", type("P", (), {"_h": None})())
    refused(_lib.PA_EINVAL, "not ordered", one, dtype=C64, op=MAX)
    refused(_lib.PA_EINVAL, "ordered comparison", one, dtype=C32, op=ANY | LT, pred=VAL)
    refused(_lib.PA_EINVAL, "unknown element type", one, dtype=9)
    refused(_lib.PA_EINVAL, "one predicate", one, op=ALL)
    refused(_lib.PA_EINVAL, "`b` is missing", one, f=DOT)
    refused(_lib.PA_EINVAL, "goes with PA_MAP_DOT only", one, f=ABS2, b=B)
    refused(_lib.PA_EINVAL, "null array pointer", one, a=None)
    refused(_lib.PA_EINVAL, "aligned to 8 bytes", one, a=C.c_void_p(0x10004))
    refused(_lib.PA_EINVAL, "aligned to 4 bytes", one, dtype=C32, f=DOT, b=C.c_void_p(0x20002))
    refused(_lib.PA_EINVAL, "`result`", one, result=None)
    refused(_lib.PA_EINVAL, "`result`", one, dtype=I32, result=C.c_void_p(0x30004))  # Int64 result
    # complex results are stored whole: ComplexF64 needs 16 bytes, ComplexF32 8
    refused(_lib.PA_EINVAL, "aligned to 16 bytes", one, dtype=C64, result=C.c_void_p(0x30008))
    refused(_lib.PA_EINVAL, "aligned to 8 bytes", one, dtype=C32, result=C.c_void_p(0x30004))
    refused(_lib.PA_EINVAL, "needs pred_value", one, op=ANY | GT)
    refused(_lib.PA_EINVAL, "negative extra dim", one, n_extra=1, extra=(-1,))
    refused(_lib.PA_EINVAL, "extra dims", one, n_extra=7, extra=(1,) * 7)
    refused(_lib.PA_EINVAL, "empty collection", empty, op=MAX, a=None)
    refused(_lib.PA_EINVAL, "empty collection", one, op=MIN, n_extra=1, extra=(0,), a=None)
    refused(_lib.PA_EINCOMPAT, "needs a communicator", four)
    assert lib.pa_launch_count() == n0


@pytest.mark.skipif(not NO_GPU, reason="a valid call runs on a machine with a GPU")
def test_valid_calls_need_a_gpu(pens):
    one, empty, _ = pens
    for kw in (dict(), dict(dtype=C64, f=ABS, op=MAX), dict(dtype=I32, f=DOT, b=B), dict(dtype=C64),
               dict(dtype=C32, result=C.c_void_p(0x30008)),
               dict(op=ANY | ISNAN), dict(dtype=C64, op=ALL | EQ, pred=(C.c_double * 2)(1, 0)),
               dict(op=ALL | GE, pred=VAL, n_extra=2, extra=(3, 2))):
        assert call(one, **kw) == _lib.PA_ENOGPU, kw
    # empty: sum / any / all are valid (0, false, true), with NULL arrays
    for op in (SUM, ANY | ISNAN, ALL | ISFINITE):
        assert call(empty, op=op, a=None) == _lib.PA_ENOGPU


def test_python_refuses_incompatible_arrays(pens):
    one, _, _ = pens
    other = pa.Pencil(one.topology, (16, 21, 41), (2, 3))
    # the checks run before anything touches device memory: plain CPU tensors stand in
    u = pa.PencilArray(one, torch.zeros(41, 21, 16, dtype=torch.float64))
    v = pa.PencilArray(other, torch.zeros(41, 21, 16, dtype=torch.float64))
    w = pa.PencilArray(one, torch.zeros(2, 41, 21, 16, dtype=torch.float64))
    z = pa.PencilArray(one, torch.zeros(41, 21, 16, dtype=torch.float32))
    with pytest.raises(pa.ArgumentError, match="same pencil"):
        pa.mapreduce(pa.realdot, "+", u, v)
    with pytest.raises(pa.ArgumentError, match="extra dims"):
        pa.mapreduce(pa.realdot, "+", u, w)
    with pytest.raises(pa.ArgumentError, match="float32"):
        pa.mapreduce(pa.realdot, "+", u, z)
    with pytest.raises(pa.ArgumentError, match="not one of the recognised"):
        pa.mapreduce(lambda x: x + 1, "+", u)
    with pytest.raises(pa.ArgumentError, match="not one of the recognised"):
        pa.any(u, "~")
    with pytest.raises(pa.ArgumentError, match="compares against"):
        pa.all(u, ">")
    with pytest.raises(pa.ArgumentError, match="one or two arrays"):
        pa.mapreduce(pa.realdot, "+", u, u, u)


def test_python_refuses_predicate_values_the_element_type_cannot_hold(pens):
    """The kernel compares in the (mapped) element type, Julia and torch in the promoted one:
    0.1 against Float32 data, 2.5 or 2^40 against Int32 data would give another Bool."""
    one, _, _ = pens
    f32 = pa.PencilArray(one, torch.zeros(41, 21, 16, dtype=torch.float32))
    i32 = pa.PencilArray(one, torch.zeros(41, 21, 16, dtype=torch.int32))
    c64 = pa.PencilArray(one, torch.zeros(41, 21, 16, dtype=torch.complex64))
    for u, pred, value, f in ((f32, ">", 0.1, None), (f32, "==", 0.1, None), (i32, "==", 2.5, None),
                              (i32, "<", 2 ** 40, None), (c64, "==", 0.1 + 1j, None),
                              (c64, ">", 0.1, abs), (f32, "<=", 1e300, None)):
        with pytest.raises(pa.ArgumentError, match="not exactly representable"):
            pa.any(u, pred, value, f=f)
        with pytest.raises(pa.ArgumentError, match="not exactly representable"):
            pa.all(u, pred, value, f=f)
    # values the element type holds exactly pass the check unchanged
    for u, value in ((f32, 0.5), (f32, float("inf")), (i32, 2.0), (i32, 7), (c64, 0.5 + 0.25j)):
        assert pa.reductions._exact(value, u.dtype)[0].item() == value
    assert math.isnan(pa.reductions._exact(float("nan"), torch.float32)[0].item())
