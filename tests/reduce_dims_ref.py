"""Reference of reductions along dims (pa_reduce_dims) for tests/test_gpu_reduce_dims.py and
tests/mp_reduce_dims_worker.py: numpy over an array in LOGICAL order, reduced dims kept with
extent 1, float sums exact per element (math.fsum) with the bound DESIGN §3l states."""
import math

import numpy as np
import torch

import pencilarrays_b200 as pa

# a bound on the roundings any one output's float sum goes through (DESIGN §3l): the members'
# sequential runs together hold at most the output's nred elements, the two team trees add at
# most 2 log2(256) and the split fold at most nred / 64, the group fold P - 1
def depth(nred, P=1):
    return nred + nred // 64 + 16 + P


def logical_view(u, t):
    """``t`` (a tensor laid out like ``u.data``, any extents) indexed in ``u``'s logical order."""
    N = len(u.space_dims)
    perm = pa.permutations.as_tuple(u.pencil.perm, N)
    v = t.permute(*reversed(range(t.dim())))
    order = list(range(v.dim()))
    for m, l in enumerate(perm):
        order[l - 1] = m
    return v.permute(*order)


def mapped(x, f, y=None):
    if f is pa.realdot:  # real(x * conj(y)), the same unfused expression as abs2
        if np.iscomplexobj(x):
            return x.real * y.real + x.imag * y.imag
        with np.errstate(over="ignore"):
            return x * y
    if f is None:
        return x
    if f is abs:
        if x.dtype == np.complex64:  # hypot of the float components, rounded once
            return np.abs(x.astype(np.complex128)).astype(np.float32)
        return np.abs(x)
    if np.iscomplexobj(x):
        return x.real * x.real + x.imag * x.imag
    with np.errstate(over="ignore"):
        return x * x  # integers wrap, as Julia's abs2


def _rows(a, dims):
    """a with the reduced axes (1-based dims) flattened last: shape (*kept, nred)."""
    red = [d - 1 for d in dims]
    kept = [i for i in range(a.ndim) if i not in red]
    b = np.transpose(a, kept + red)
    return b.reshape(b.shape[:len(kept)] + (-1,))


def _keep(r, shape, dims):
    s = list(shape)
    for d in dims:
        s[d - 1] = 1
    return r.reshape(s)


def jl_max(a, axis):
    """Julia's maximum along the last axis: NaN wins, -0.0 < 0.0."""
    out = np.max(a, axis=axis) if a.shape[axis] else np.empty(a.shape[:-1], a.dtype)
    if np.issubdtype(a.dtype, np.floating) and a.size:
        # max picks 0.0 over -0.0 only if a +0.0 is present
        zero = out == 0
        has_pos = np.any((a == 0) & ~np.signbit(a), axis=axis)
        out = np.where(zero & ~has_pos, -0.0, np.where(zero, 0.0, out)).astype(a.dtype)
        out = np.where(np.any(np.isnan(a), axis=axis), np.nan, out).astype(a.dtype)
    return out


def jl_min(a, axis):
    out = np.min(a, axis=axis) if a.shape[axis] else np.empty(a.shape[:-1], a.dtype)
    if np.issubdtype(a.dtype, np.floating) and a.size:
        zero = out == 0
        has_neg = np.any((a == 0) & np.signbit(a), axis=axis)
        out = np.where(zero & has_neg, -0.0, np.where(zero, 0.0, out)).astype(a.dtype)
        out = np.where(np.any(np.isnan(a), axis=axis), np.nan, out).astype(a.dtype)
    return out


PRED = {"==": np.equal, "!=": np.not_equal, "<": np.less, "<=": np.less_equal, ">": np.greater,
        ">=": np.greater_equal}


def expect(x, f, op, dims, pred=None, value=None, y=None):
    """(want, tol) in logical order; tol None: exact.  x (and y, the second array of realdot):
    numpy arrays in logical order."""
    fx = mapped(x, f, y)
    rows = _rows(fx, dims)
    if op in ("any", "all"):
        if pred == "isnan":
            hit = np.isnan(rows)
        elif pred == "isfinite":
            hit = np.isfinite(rows)
        else:
            hit = PRED[pred](rows, value)
        r = hit.any(axis=-1) if op == "any" else hit.all(axis=-1)
        return _keep(r, x.shape, dims), None
    if op == "max":
        return _keep(jl_max(rows, -1), x.shape, dims), None
    if op == "min":
        return _keep(jl_min(rows, -1), x.shape, dims), None
    if np.issubdtype(rows.dtype, np.integer):
        acc = rows.astype(np.int64).sum(axis=-1) if rows.dtype == np.int32 else rows.sum(axis=-1)
        return _keep(acc, x.shape, dims), None
    flat = rows.reshape(-1, rows.shape[-1])
    cplx = np.iscomplexobj(flat)
    want = np.empty(flat.shape[0], np.complex128 if cplx else np.float64)
    tol = np.empty(flat.shape[0])
    for i, row in enumerate(flat):
        if cplx:
            want[i] = complex(math.fsum(row.real.astype(np.float64)), math.fsum(row.imag.astype(np.float64)))
        else:
            want[i] = math.fsum(row.astype(np.float64))
        tol[i] = math.fsum(np.abs(row.astype(np.complex128 if cplx else np.float64)))
    n = rows.shape[-1]
    single = rows.dtype in (np.float32, np.complex64)
    eps = 2.0 ** -53
    tol = depth(n) * eps * tol + (np.abs(want) * 2.0 ** -24 if single else 0.0)
    return _keep(want, x.shape, dims), _keep(tol, x.shape, dims)


def check(got, want, tol, what):
    """got: numpy result in logical order."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if tol is None:
        if np.issubdtype(want.dtype, np.floating) or np.iscomplexobj(want):
            ok = (got == want) | (np.isnan(got) & np.isnan(want))
            ok &= np.signbit(np.real(got)) == np.signbit(np.real(want))
            assert ok.all(), (what, got[~ok][:4], want[~ok][:4])
        else:
            assert np.array_equal(got.astype(want.dtype), want), (what, got, want)
    else:
        err = np.abs(got.astype(want.dtype) - want)
        assert (err <= tol + 1e-300).all(), (what, err.max(), tol.min())
