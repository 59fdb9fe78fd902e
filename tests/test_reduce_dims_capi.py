"""pa_reduce_dims on the host (no GPU needed): every refusal in the order pa_b200.h states it,
PA_ENOGPU for valid calls on a machine without a GPU, result types as pa_reduce_result_type gives
them, and the Python mirror's ``dims`` checks and result shapes."""
import ctypes as C
import itertools

import pytest
import torch

import pencilarrays_b200 as pa
from pencilarrays_b200 import _lib
from pencilarrays_b200._lib import lib, i64arr
from pencilarrays_b200.reductions import result_shape

F64, F32, C64, C32, I32, I64 = range(6)
ID, ABS, ABS2, DOT = range(4)
SUM, MAX, MIN, ANY, ALL = range(5)
NO_GPU = lib.pa_device_count() == 0
BUF = (C.c_double * 64)()
P = C.cast(BUF, C.c_void_p)


def pencil(size, grid=(1, 1), decomp=(2, 3), perm=None):
    kw = {"permute": pa.Permutation(*perm)} if perm else {}
    comm = pa.COMM_SELF if grid == (1, 1) else pa.Comm(0, grid[0] * grid[1])
    return pa.Pencil(pa.MPITopology(comm, grid), size, decomp, **kw)


def call(pen, dims, extra=(), dtype=F64, f=ID, op=SUM, a=P, b=None, result=P, pred=None):
    arr = (C.c_int * max(1, len(dims)))(*dims) if dims is not None else None
    return lib.pa_reduce_dims(pen._h, len(extra), i64arr(extra) if extra else None, None, dtype, f,
                              op, pred, a, b, len(dims) if dims is not None else 0, arr, result,
                              None)


def err():
    return lib.pa_last_error().decode()


def test_export_and_signature():
    assert hasattr(lib, "pa_reduce_dims")
    assert "pa_reduce_dims" in _lib.SIGNATURES


def test_refusals_in_order():
    pen = pencil((4, 3, 2))
    assert lib.pa_reduce_dims(None, 0, None, None, F64, ID, SUM, None, P, None, 1,
                              (C.c_int * 1)(1), P, None) == _lib.PA_EINVAL
    assert "null pencil" in err()
    # pa_reduce's result-type refusal comes before the dims
    assert call(pen, (9,), dtype=C64, op=MAX) == _lib.PA_EINVAL and "not ordered" in err()
    assert call(pen, (1,), extra=(-1,)) == _lib.PA_EINVAL and "negative extra dim" in err()
    for dims, what in (((), "at least one"), (None, "at least one"), ((0,), "out of range"),
                       ((4,), "out of range"), ((1, 5), "out of range"), ((2, 2), "twice"),
                       ((3, 1, 3), "twice")):
        assert call(pen, dims) == _lib.PA_EINVAL, dims
        assert err().startswith("pa_reduce_dims:") and what in err(), (dims, err())
    # extra dims count after the spatial ones: dim 4 of a pencil with one extra dim is valid
    if NO_GPU:  # (with a GPU the valid call would run on these host stand-ins)
        assert call(pen, (4,), extra=(2,)) == _lib.PA_ENOGPU
    assert call(pen, (5,), extra=(2,)) == _lib.PA_EINVAL and "out of range 1..4" in err()
    # bad dims come before the array checks
    assert call(pen, (0,), a=None) == _lib.PA_EINVAL and "out of range" in err()
    assert call(pen, (1,), b=P) == _lib.PA_EINVAL and "PA_MAP_DOT only" in err()
    assert call(pen, (1,), f=DOT) == _lib.PA_EINVAL and "`b` is missing" in err()
    assert call(pen, (1,), a=None) == _lib.PA_EINVAL and "null array pointer" in err()
    assert call(pen, (1,), result=None) == _lib.PA_EINVAL and "`result`" in err()
    assert call(pen, (1,), op=ANY | _lib.PA_PRED_GT) == _lib.PA_EINVAL and "pred_value" in err()


def test_empty_reduced_ranges():
    pen = pencil((4, 0, 2))
    # max / min over a globally empty reduced range are refused, a sum is not
    for op in (MAX, MIN):
        assert call(pen, (2,), op=op) == _lib.PA_EINVAL and "empty collection" in err()
        assert call(pen, (1, 2), op=op) == _lib.PA_EINVAL
        # the reduced range is not empty: the (empty) result is fine, and so a NULL result
        want = _lib.PA_ENOGPU if NO_GPU else _lib.PA_OK
        if NO_GPU:
            assert call(pen, (1, 3), op=op, a=None, result=None) == want
    if NO_GPU:
        assert call(pen, (2,), op=SUM) == _lib.PA_ENOGPU


def test_capacity_and_communicator():
    # a 1 x 2 grid without a communicator: the capacity refusal (decided from the global geometry,
    # the largest local result on any rank) comes before the communicator's
    big = pencil((1030, 520, 4), grid=(1, 2), decomp=(2, 3))
    assert call(big, (3,)) == _lib.PA_EINVAL and "partial area" in err()
    assert call(big, (1, 2)) == _lib.PA_EINCOMPAT and "needs a communicator" in err()
    # one rank: no window, no capacity limit
    one = pencil((1030, 520, 4))
    if NO_GPU:
        assert call(one, (3,)) == _lib.PA_ENOGPU


@pytest.mark.skipif(not NO_GPU, reason="on a GPU machine valid calls run (tests/test_gpu_reduce_dims.py)")
def test_valid_calls_need_a_gpu():
    pen = pencil((4, 3, 2), perm=(2, 1, 3))
    for dims in itertools.chain.from_iterable(itertools.combinations(range(1, 5), k) for k in (1, 2, 3, 4)):
        for dtype, f, op in ((F64, ID, SUM), (C32, ABS, MAX), (I32, ABS2, SUM), (C64, DOT, SUM),
                             (I64, ID, ALL | _lib.PA_PRED_ISFINITE)):
            b = P if f == DOT else None
            assert call(pen, dims, extra=(2,), dtype=dtype, f=f, op=op, b=b) == _lib.PA_ENOGPU, dims


def test_result_types_follow_pa_reduce_result_type():
    """pa_reduce_dims accepts exactly the (dtype, map, op) combinations pa_reduce_result_type
    gives a type for, and names itself when it refuses one.  (The GPU tests check that the
    mirror's result has that type.)"""
    pen = pencil((4, 3, 2))
    preds = [k << 4 for k in range(1, 9)]
    ops = [SUM, MAX, MIN] + [b | p for b in (ANY, ALL) for p in preds] + [ANY, SUM | (1 << 4)]
    val = (C.c_double * 2)(0.0, 0.0)
    for dtype, f, op in itertools.product(range(6), range(4), ops):
        rt = C.c_int(-1)
        ok = lib.pa_reduce_result_type(dtype, f, op, C.byref(rt)) == _lib.PA_OK
        if ok and not NO_GPU:
            continue  # (with a GPU the valid call would run on these host stand-ins)
        s = call(pen, (1,), dtype=dtype, f=f, op=op, b=P if f == DOT else None,
                 pred=C.cast(val, C.c_void_p))
        if not ok:
            assert s == _lib.PA_EINVAL and err().startswith("pa_reduce_dims: dtype"), (dtype, f, op)
        elif NO_GPU:
            assert s == _lib.PA_ENOGPU, (dtype, f, op, err())


@pytest.mark.parametrize("perm,extra", [(None, ()), ((2, 1, 3), (2,)), ((3, 2, 1), (3, 2)),
                                        ((3, 1, 2), (1,))])
def test_python_result_shapes(perm, extra):
    pen = pencil((5, 6, 7), perm=perm)
    mem = pa.size_local(pen, pa.MemoryOrder())
    data = torch.empty(tuple(reversed(mem + extra)))  # host tensor: only the shape is read
    u = pa.PencilArray(pen, data, extra)
    N = 3
    p = pa.permutations.as_tuple(pen.perm, N)
    for k in range(1, N + len(extra) + 1):
        for dims in itertools.combinations(range(1, N + len(extra) + 1), k):
            for order in (dims, tuple(reversed(dims))):
                got_dims, shape = result_shape(u, order)
                assert got_dims == order
                # the shape of u.data with every reduced position 1
                want = list(data.shape)
                for d in dims:
                    m = p.index(d) if d <= N else d - 1  # memory dim
                    want[len(want) - 1 - m] = 1
                assert shape == tuple(want), (perm, extra, order)
                # and in logical order: 1 along the reduced dims, the local size elsewhere
                lg = [mem[p.index(l)] if l <= N else extra[l - N - 1] for l in range(1, N + len(extra) + 1)]
                jl = tuple(reversed(shape))
                for l in range(1, N + len(extra) + 1):
                    m = p.index(l) if l <= N else l - 1
                    assert jl[m] == (1 if l in dims else lg[l - 1])
    assert result_shape(u, 2)[0] == (2,)


def test_python_dims_validation():
    pen = pencil((5, 6, 7))
    u = pa.PencilArray(pen, torch.empty((2, 7, 6, 5)), (2,))
    for bad in ((), (0,), (5,), (1, 1), ("x",), (1.0,), (True,), None.__class__):
        with pytest.raises(pa.ArgumentError):
            result_shape(u, bad)
    assert result_shape(u, [4, 1])[1] == (1, 7, 6, 1)
