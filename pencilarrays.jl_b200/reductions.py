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

Every function takes ``dims``: ``None`` (the default) reduces over everything, as above; a dim or
a collection of 1-based LOGICAL dims (``1..N`` the pencil's spatial dims, ``N+1..`` its extra
dims) reduces over those only (``pa_reduce_dims``, DESIGN §3l).  The result is then a tensor of
``u.data.shape`` with every reduced position set to 1: along each kept dim it holds this rank's
local range, combined over the ranks that share it, so ``u.data - mean`` broadcasts with no
further exchange.
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
from .permutations import as_tuple
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


def result_shape(u: PencilArray, dims):
    """The checked ``dims`` as a tuple of 1-based logical dims, and the torch shape of the result
    of a reduction of ``u`` along them: ``u.data.shape`` with the reduced positions set to 1."""
    if isinstance(dims, int) and not isinstance(dims, bool):
        dims = (dims,)
    try:
        dims = tuple(dims)
    except TypeError:
        raise ArgumentError(_lib.PA_EINVAL, f"dims {dims!r} is not a dim or a collection of dims") from None
    N, nd = len(u.space_dims), u.data.dim()
    if not dims:
        raise ArgumentError(_lib.PA_EINVAL, "dims must name at least one dim")
    for d in dims:
        if not isinstance(d, int) or isinstance(d, bool) or not 1 <= d <= nd:
            raise ArgumentError(_lib.PA_EINVAL, f"dim {d!r} out of range 1..{nd} ({N} spatial dims, "
                                f"then {nd - N} extra)")
    if len(set(dims)) != len(dims):
        raise ArgumentError(_lib.PA_EINVAL, f"dims {dims} name a dim twice")
    perm = as_tuple(u.pencil.perm, N)  # memory dim m holds logical dim perm[m]
    shape = list(u.data.shape)
    for d in dims:
        m = perm.index(d) if d <= N else d - 1
        shape[nd - 1 - m] = 1
    return dims, tuple(shape)


def _reduce(code_map, code_op, u: PencilArray, vs, value=None, dims=None):
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
    comm = u.pencil.topology.comm
    ex = u.extra_dims
    args = (u.pencil._h, len(ex), i64arr(ex), comm.handle, dt, code_map, code_op,
            C.c_void_p(pred.data_ptr()) if pred is not None else None,
            C.c_void_p(u.data_ptr() or None), C.c_void_p(vs[0].data_ptr() or None) if vs else None)
    if dims is None:
        result = torch.empty((), dtype=_TORCH[out.value], device=u.data.device)
        with torch.cuda.device(u.data.device):
            check(lib.pa_reduce(*args, C.c_void_p(result.data_ptr()), _stream_ptr()))
        return result
    dims, shape = result_shape(u, dims)
    result = torch.empty(shape, dtype=_TORCH[out.value], device=u.data.device)
    with torch.cuda.device(u.data.device):
        check(lib.pa_reduce_dims(*args, len(dims), (C.c_int * len(dims))(*dims),
                                 C.c_void_p(result.data_ptr() or None), _stream_ptr()))
    return result


def mapreduce(f, op, u: PencilArray, *vs: PencilArray, dims=None):
    """``mapreduce(f, op, u, vs...; dims)`` over all ranks; ``f`` of two arrays is :func:`realdot`."""
    return _reduce(_lookup(_MAPS, f, "function"), _lookup(_OPS, op, "op"), u, vs, dims=dims)


def sum(u: PencilArray, f=None, dims=None):
    """``sum(f, u; dims)``."""
    return mapreduce(f, "+", u, dims=dims)


def maximum(u: PencilArray, f=None, dims=None):
    """``maximum(f, u; dims)``; a NaN anywhere gives NaN.  Refused for a globally empty range."""
    return mapreduce(f, "max", u, dims=dims)


def minimum(u: PencilArray, f=None, dims=None):
    """``minimum(f, u; dims)``; a NaN anywhere gives NaN.  Refused for a globally empty range."""
    return mapreduce(f, "min", u, dims=dims)


def _pred(op, u, pred, value, f, dims):
    p = _lookup(_PREDS, pred, "predicate")
    if p in (_lib.PA_PRED_ISNAN, _lib.PA_PRED_ISFINITE):
        value = None
    elif value is None:
        raise ArgumentError(_lib.PA_EINVAL, f"the predicate {pred!r} compares against `value`")
    return _reduce(_lookup(_MAPS, f, "function"), op | p, u, (), value, dims)


def any(u: PencilArray, pred, value=None, f=None, dims=None):
    """``any(x -> pred(f(x), value), u; dims)``, e.g. ``any(u, ">", 0)`` or ``any(u, "isnan")``."""
    return _pred(_lib.PA_OP_ANY, u, pred, value, f, dims)


def all(u: PencilArray, pred, value=None, f=None, dims=None):
    """``all(x -> pred(f(x), value), u; dims)``, e.g. ``all(u, "isfinite")``."""
    return _pred(_lib.PA_OP_ALL, u, pred, value, f, dims)


def _spectrum_geometry(u: PencilArray, rfft_dim, rfft_n, scales, width):
    N = len(u.space_dims)
    rd = 0 if rfft_dim is None else rfft_dim
    if not isinstance(rd, int) or isinstance(rd, bool):
        raise ArgumentError(_lib.PA_EINVAL, f"rfft_dim {rfft_dim!r} is not a dim")
    rn = 0 if rfft_n is None else rfft_n
    if not isinstance(rn, int) or isinstance(rn, bool):
        raise ArgumentError(_lib.PA_EINVAL, f"rfft_n {rfft_n!r} is not an integer")
    sc = None
    if scales is not None:
        try:
            sc = tuple(float(x) for x in scales)
        except (TypeError, ValueError):
            raise ArgumentError(_lib.PA_EINVAL, f"scales {scales!r} are not {N} numbers") from None
        if len(sc) != N:
            raise ArgumentError(_lib.PA_EINVAL, f"scales {scales!r}: one per spatial dim ({N})")
        sc = (C.c_double * N)(*sc)
    try:
        width = float(width)
    except (TypeError, ValueError):
        raise ArgumentError(_lib.PA_EINVAL, f"width {width!r} is not a number") from None
    return rd, rn, sc, width


def _dim_list(u: PencilArray, dims, what, spatial):
    """``dims`` (a dim or a collection of 1-based logical dims) checked as :func:`result_shape`
    checks them, as a tuple: spatial dims only for the bin dims, any dim for the kept ones."""
    if isinstance(dims, int) and not isinstance(dims, bool):
        dims = (dims,)
    try:
        dims = tuple(dims)
    except TypeError:
        raise ArgumentError(_lib.PA_EINVAL, f"{what} {dims!r} is not a dim or a collection of dims") from None
    N, nd = len(u.space_dims), u.data.dim()
    top = N if spatial else nd
    for d in dims:
        if not isinstance(d, int) or isinstance(d, bool) or not 1 <= d <= top:
            raise ArgumentError(_lib.PA_EINVAL, f"{what}: dim {d!r} out of range 1..{top} "
                                + ("(the spatial dims)" if spatial else
                                   f"({N} spatial dims, then {nd - N} extra)"))
    if len(set(dims)) != len(dims):
        raise ArgumentError(_lib.PA_EINVAL, f"{what} {dims} name a dim twice")
    return dims


def _bin_dims(u: PencilArray, dims):
    """The checked bin dims (None: every spatial dim)."""
    if dims is None:
        dims = tuple(range(1, len(u.space_dims) + 1))
    dims = _dim_list(u, dims, "dims", True)
    if not dims:
        raise ArgumentError(_lib.PA_EINVAL, "dims must name at least one bin dim")
    return dims


def spectrum_nbins(u: PencilArray, *, rfft_dim=None, rfft_n=None, scales=None, width=1.0, dims=None):
    """The default bin count of :func:`shell_spectrum`: the bin of the extreme mode over the bin
    dims ``dims`` (default: every spatial dim) plus one, as the library computes it
    (``pa_shell_spectrum_nbins`` / ``pa_shell_spectrum_dims_nbins``)."""
    rd, rn, sc, width = _spectrum_geometry(u, rfft_dim, rfft_n, scales, width)
    out = C.c_int()
    if dims is None:
        check(lib.pa_shell_spectrum_nbins(u.pencil._h, rd, rn, sc, width, C.byref(out)))
    else:
        bd = _bin_dims(u, dims)
        check(lib.pa_shell_spectrum_dims_nbins(u.pencil._h, rd, rn, sc, width, len(bd),
                                               (C.c_int * len(bd))(*bd), C.byref(out)))
    return out.value


def shell_spectrum(u: PencilArray, v: PencilArray = None, *, rfft_dim=None, rfft_n=None,
                   scales=None, width=1.0, nbins=None, dims=None, keep=None):
    """Shell-binned spectrum ``E(b) = sum over bin(|k|) == b of w * abs2(u)`` (with ``v``: of
    ``w * real(u * conj(v))``, a co-spectrum) of complex arrays whose spatial dims hold the modes
    of an unnormalised DFT (``pa_shell_spectrum``, DESIGN §3m).  ``rfft_dim``: the 1-based logical
    dim holding the ``n // 2 + 1`` bins of a real-to-complex transform of length ``rfft_n``
    (default ``2 (M - 1)``), whose interior bins count twice; ``scales``: one wavenumber scale per
    spatial dim (``2 pi / L``; default 1); ``width``: the shell width; ``nbins``: default
    :func:`spectrum_nbins`.  Extra dims add into the same bins.  Returns the global spectrum (the
    same bits on every rank), a 1-d tensor of ``nbins`` float64 (float32 for complex64 arrays) on
    ``u``'s device, computed on torch's current stream in one kernel per rank.

    ``dims`` and ``keep`` (``pa_shell_spectrum_dims``, DESIGN §3n): ``|k|`` is formed from the bin
    dims ``dims`` only (1-based spatial dims; default every one), each dim in ``keep`` (1-based
    logical dims, extra dims ``N+1..`` included, none a bin dim) is kept, and every other dim is
    summed into the bins: ``dims=(1, 3), keep=(2,)`` is E(k_h; y), ``dims=(1,)`` E(k_x), and
    ``keep=(4,)`` on a 3-component field the per-component spectra.  With ``keep`` the result has
    ``u.data.shape`` with every non-kept position set to 1 and a trailing ``nbins`` dim; along each
    kept dim it holds this rank's local range, combined over the ranks that share it.  Without
    ``keep`` it is ``(nbins,)``."""
    if not isinstance(u, PencilArray):
        raise ArgumentError(_lib.PA_EINVAL, "shell_spectrum takes PencilArrays")
    if v is not None:
        if not isinstance(v, PencilArray) or v.pencil is not u.pencil:
            raise ArgumentError(_lib.PA_EINVAL, "arrays are not compatible: not on the same pencil")
        if v.extra_dims != u.extra_dims:
            raise ArgumentError(_lib.PA_EINVAL, "arrays are not compatible: extra dims "
                                f"{v.extra_dims} != {u.extra_dims}")
        if v.dtype != u.dtype:
            raise ArgumentError(_lib.PA_EINVAL, f"arrays are not compatible: {v.dtype} != {u.dtype}")
    if u.dtype not in _REAL:
        raise ArgumentError(_lib.PA_EINVAL, f"a spectrum is of complex arrays, not {u.dtype}")
    sub = dims is not None or keep is not None
    who = "pa_shell_spectrum_dims" if sub else "pa_shell_spectrum"
    shape = None
    if sub:
        bd = _bin_dims(u, dims)
        kd = () if keep is None else _dim_list(u, keep, "keep", False)
        both = set(bd) & set(kd)
        if both:
            raise ArgumentError(_lib.PA_EINVAL, f"dim {min(both)} is both a bin dim and a kept dim")
        if kd:
            red = tuple(d for d in range(1, u.data.dim() + 1) if d not in kd)
            shape = result_shape(u, red)[1]
    rd, rn, sc, width = _spectrum_geometry(u, rfft_dim, rfft_n, scales, width)
    out = C.c_int()  # (the geometry's checks, before anything is allocated)
    if sub:
        check(lib.pa_shell_spectrum_dims_nbins(u.pencil._h, rd, rn, sc, width, len(bd),
                                               (C.c_int * len(bd))(*bd), C.byref(out)))
    else:
        check(lib.pa_shell_spectrum_nbins(u.pencil._h, rd, rn, sc, width, C.byref(out)))
    if nbins is None:
        nbins = out.value
    if not isinstance(nbins, int) or isinstance(nbins, bool) or \
            not 1 <= nbins <= _lib.PA_SPECTRUM_MAX_BINS:
        raise ArgumentError(_lib.PA_EINVAL, f"{who}: nbins {nbins!r} out of range "
                            f"1..{_lib.PA_SPECTRUM_MAX_BINS}")
    code_map = _lib.PA_MAP_ABS2 if v is None else _lib.PA_MAP_DOT
    dt = _DTYPES[u.dtype]
    result = torch.empty((nbins,) if shape is None else shape + (nbins,), dtype=_REAL[u.dtype],
                         device=u.data.device)
    ex = u.extra_dims
    args = (u.pencil._h, len(ex), i64arr(ex), u.pencil.topology.comm.handle, dt, code_map,
            C.c_void_p(u.data_ptr() or None),
            C.c_void_p(v.data_ptr() or None) if v is not None else None, rd, rn, sc, width, nbins)
    with torch.cuda.device(u.data.device):
        if sub:
            check(lib.pa_shell_spectrum_dims(*args, len(bd), (C.c_int * len(bd))(*bd), len(kd),
                                             (C.c_int * max(1, len(kd)))(*kd),
                                             C.c_void_p(result.data_ptr() or None), _stream_ptr()))
        else:
            check(lib.pa_shell_spectrum(*args, C.c_void_p(result.data_ptr() or None), _stream_ptr()))
    return result
