"""Global reductions over PencilArrays (src/reductions.jl:10-38): ``mapreduce`` / ``sum`` /
``maximum`` / ``minimum`` / ``any`` / ``all`` over ``parent(u)`` (extra dims included), combined
across every rank of the array's communicator.  Each call is ONE kernel per rank
(``pa_reduce``), runs on torch's current stream without synchronising the host, and returns the
global result on every rank as a 0-d tensor on the array's device.

Recognised functions (anything else is refused; the library has no generic fallback):
``f``: ``None`` / ``identity``, ``abs`` (the builtin), :func:`abs2`, and for two arrays
:func:`realdot` = ``real(x * conj(y))``; ``op``: ``"+"`` / ``operator.add``, ``max``, ``min``;
predicates of ``any`` / ``all``: ``"=="``, ``"!="``, ``"<"``, ``"<="``, ``">"``, ``">="``
against ``value`` (which must be exactly representable in the mapped element type: the
comparison runs in that type), or ``"isnan"`` / ``"isfinite"``.  The result's type comes from the library
(``pa_reduce_result_type``): sum of int32 gives int64, abs / abs2 / realdot of complex values
the real type, any / all bool.
"""
from __future__ import annotations

import builtins
import ctypes as C
import math
import operator

import torch

from . import _lib
from ._lib import lib, check, i64arr, ArgumentError
from .arrays import PencilArray
from .transpositions import _stream_ptr


def identity(x):
    return x


def abs2(x):
    """``abs2(x)``: ``x * x`` for reals (integers wrap), ``re^2 + im^2`` for complex values."""
    return (x * x.conjugate()).real if isinstance(x, complex) else x * x


def realdot(x, y):
    """``real(x * conj(y))``: the map of ``mapreduce(realdot, +, u, v)`` (an inner product)."""
    return (x * complex(y).conjugate()).real if isinstance(x, complex) else x * y


_DTYPES = {torch.float64: _lib.PA_FLOAT64, torch.float32: _lib.PA_FLOAT32,
           torch.complex128: _lib.PA_COMPLEXF64, torch.complex64: _lib.PA_COMPLEXF32,
           torch.int32: _lib.PA_INT32, torch.int64: _lib.PA_INT64}
_TORCH = {v: k for k, v in _DTYPES.items()}
_TORCH[_lib.PA_BOOL] = torch.bool
_REAL = {torch.complex128: torch.float64, torch.complex64: torch.float32}

_MAPS = {None: _lib.PA_MAP_IDENTITY, identity: _lib.PA_MAP_IDENTITY, "identity": _lib.PA_MAP_IDENTITY,
         builtins.abs: _lib.PA_MAP_ABS, "abs": _lib.PA_MAP_ABS, abs2: _lib.PA_MAP_ABS2,
         "abs2": _lib.PA_MAP_ABS2, realdot: _lib.PA_MAP_DOT, "realdot": _lib.PA_MAP_DOT}
_OPS = {"+": _lib.PA_OP_SUM, operator.add: _lib.PA_OP_SUM, builtins.max: _lib.PA_OP_MAX,
        "max": _lib.PA_OP_MAX, builtins.min: _lib.PA_OP_MIN, "min": _lib.PA_OP_MIN}
_PREDS = {"==": _lib.PA_PRED_EQ, operator.eq: _lib.PA_PRED_EQ, "!=": _lib.PA_PRED_NE,
          operator.ne: _lib.PA_PRED_NE, "<": _lib.PA_PRED_LT, operator.lt: _lib.PA_PRED_LT,
          "<=": _lib.PA_PRED_LE, operator.le: _lib.PA_PRED_LE, ">": _lib.PA_PRED_GT,
          operator.gt: _lib.PA_PRED_GT, ">=": _lib.PA_PRED_GE, operator.ge: _lib.PA_PRED_GE,
          "isnan": _lib.PA_PRED_ISNAN, math.isnan: _lib.PA_PRED_ISNAN,
          "isfinite": _lib.PA_PRED_ISFINITE, math.isfinite: _lib.PA_PRED_ISFINITE}


def _lookup(table, key, what):
    try:
        return table[key]
    except (KeyError, TypeError):
        raise ArgumentError(_lib.PA_EINVAL, f"{what} {key!r} is not one of the recognised ones") from None


def result_dtype(dtype: torch.dtype, f=None, op="+"):
    """The result's torch dtype of ``mapreduce(f, op, ...)`` on ``dtype`` arrays, as the library
    decides it (``pa_reduce_result_type``)."""
    out = C.c_int()
    code = op if isinstance(op, int) else _lookup(_OPS, op, "op")
    check(lib.pa_reduce_result_type(_lookup(_DTYPES, dtype, "element type"),
                                    _lookup(_MAPS, f, "function"), code, C.byref(out)))
    return _TORCH[out.value]


def _exact(value, vt):
    """``value`` as a one-element tensor of the mapped type ``vt``, refused unless it converts
    exactly: the kernel compares in ``vt``, Julia and torch in the promoted type, and the two
    agree only for values ``vt`` holds exactly (``any(u_float32, ">", 0.1)`` would otherwise
    compare against 0.1f0)."""
    try:
        t = torch.tensor(value, dtype=vt).reshape(1)
        back = t[0].item()
        same = back == value or (back != back and value != value)  # NaN stays NaN
    except (TypeError, ValueError, RuntimeError, OverflowError):
        same = False
    if not same:
        raise ArgumentError(_lib.PA_EINVAL, f"the predicate's value {value!r} is not exactly "
                            f"representable as {vt}; compare against a value of that type")
    return t


def _reduce(code_map, code_op, u: PencilArray, vs, value=None):
    if len(vs) > 1:
        raise ArgumentError(_lib.PA_EINVAL, f"mapreduce takes one or two arrays: got {1 + len(vs)}")
    for v in vs:  # _check_compatible_arrays (arrays.jl:499-504), plus what the kernel reads
        if not isinstance(v, PencilArray) or v.pencil is not u.pencil:
            raise ArgumentError(_lib.PA_EINVAL, "arrays are not compatible: not on the same pencil")
        if v.extra_dims != u.extra_dims:
            raise ArgumentError(_lib.PA_EINVAL, "arrays are not compatible: extra dims "
                                f"{v.extra_dims} != {u.extra_dims}")
        if v.dtype != u.dtype:
            raise ArgumentError(_lib.PA_EINVAL, f"arrays are not compatible: {v.dtype} != {u.dtype}")
    dt = _lookup(_DTYPES, u.dtype, "element type")
    out = C.c_int()
    check(lib.pa_reduce_result_type(dt, code_map, code_op, C.byref(out)))
    pred = None
    if value is not None:  # one value of the mapped type
        vt = u.dtype if code_map == _lib.PA_MAP_IDENTITY else _REAL.get(u.dtype, u.dtype)
        pred = _exact(value, vt)
    result = torch.empty((), dtype=_TORCH[out.value], device=u.data.device)
    comm = u.pencil.topology.comm
    ex = u.extra_dims
    with torch.cuda.device(u.data.device):
        check(lib.pa_reduce(u.pencil._h, len(ex), i64arr(ex), comm.handle, dt, code_map, code_op,
                            C.c_void_p(pred.data_ptr()) if pred is not None else None,
                            C.c_void_p(u.data_ptr() or None),
                            C.c_void_p(vs[0].data_ptr() or None) if vs else None,
                            C.c_void_p(result.data_ptr()), _stream_ptr()))
    return result


def mapreduce(f, op, u: PencilArray, *vs: PencilArray):
    """``mapreduce(f, op, u, vs...)`` over all ranks; ``f`` of two arrays is :func:`realdot`."""
    return _reduce(_lookup(_MAPS, f, "function"), _lookup(_OPS, op, "op"), u, vs)


def sum(u: PencilArray, f=None):
    """``sum(f, u)``."""
    return mapreduce(f, "+", u)


def maximum(u: PencilArray, f=None):
    """``maximum(f, u)``; a NaN anywhere gives NaN.  Refused for a globally empty array."""
    return mapreduce(f, "max", u)


def minimum(u: PencilArray, f=None):
    """``minimum(f, u)``; a NaN anywhere gives NaN.  Refused for a globally empty array."""
    return mapreduce(f, "min", u)


def _pred(op, u, pred, value, f):
    p = _lookup(_PREDS, pred, "predicate")
    if p in (_lib.PA_PRED_ISNAN, _lib.PA_PRED_ISFINITE):
        value = None
    elif value is None:
        raise ArgumentError(_lib.PA_EINVAL, f"the predicate {pred!r} compares against `value`")
    return _reduce(_lookup(_MAPS, f, "function"), op | p, u, (), value)


def any(u: PencilArray, pred, value=None, f=None):
    """``any(x -> pred(f(x), value), u)``, e.g. ``any(u, ">", 0)`` or ``any(u, "isnan")``."""
    return _pred(_lib.PA_OP_ANY, u, pred, value, f)


def all(u: PencilArray, pred, value=None, f=None):
    """``all(x -> pred(f(x), value), u)``, e.g. ``all(u, "isfinite")``."""
    return _pred(_lib.PA_OP_ALL, u, pred, value, f)
