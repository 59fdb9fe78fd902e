"""NumPy reference of spectra over chosen dims (pa_shell_spectrum_dims, DESIGN §3n) for the tests:
bins over the bin dims only (each operation correctly rounded, so they match the library bit for
bit), Hermitian weights along the r2c dim whatever its role, per (kept index, bin) math.fsum of the
contributions and of their absolute values, the default bin count and the rounding bound."""
import math

import numpy as np

import spectrum_ref as R


def shells(size, dims, rfft_dim=None, scales=None, width=1.0):
    """floor(sqrt(q) / width + 0.5) of every mode, q over the bin dims `dims` (1-based) in logical
    order: an fp64 array of `size` in logical order."""
    N = len(size)
    scales = scales or (1.0,) * N
    q = np.zeros(size)
    for d in range(N):
        if d + 1 not in dims:
            continue
        k = scales[d] * R.wavenumbers(size[d], rfft_dim == d + 1).astype(np.float64)
        sh = [1] * N
        sh[d] = size[d]
        q = q + (k * k).reshape(sh)
    return np.floor(np.sqrt(q) / width + 0.5)


def default_nbins(size, dims, rfft_dim=None, scales=None, width=1.0):
    N = len(size)
    scales = scales or (1.0,) * N
    q = 0.0
    for d in range(N):
        if d + 1 not in dims:
            continue
        top = 0 if size[d] == 0 else size[d] - 1 if rfft_dim == d + 1 else size[d] // 2
        k = scales[d] * float(top)
        q = q + k * k
    return int(math.floor(math.sqrt(q) / width + 0.5)) + 1


def spectrum(x, N, nbins, dims, keep=(), y=None, rfft_dim=None, rfft_n=None, scales=None,
             width=1.0):
    """(exact, abs_sum) of shape (the kept dims' global extents in logical order) + (nbins,) (NaN:
    the value holds a NaN): x (and y) in logical order, the N spatial dims first, extra dims last."""
    size = x.shape[:N]
    pad = (1,) * (x.ndim - N)
    b = np.broadcast_to(shells(size, dims, rfft_dim, scales, width).reshape(size + pad), x.shape)
    w = R.mode_weights(size, rfft_dim, rfft_n).reshape(size + pad)
    c = R.contributions(x, y) * w
    kept = [d - 1 for d in keep]
    rest = [i for i in range(x.ndim) if i not in kept]
    kshape = tuple(x.shape[i] for i in kept)
    nk = int(np.prod(kshape))
    c = np.transpose(c, kept + rest).reshape(nk, -1)
    b = np.transpose(b, kept + rest).reshape(nk, -1)
    exact = np.zeros((nk, nbins))
    absum = np.zeros((nk, nbins))
    for o in range(nk):
        order = np.argsort(b[o], kind="stable")
        bs, cs = b[o][order], c[o][order]
        cuts = np.searchsorted(bs, np.arange(nbins + 1))
        for k in range(nbins):
            sel = cs[cuts[k]:cuts[k + 1]]
            if np.isnan(sel).any():
                exact[o, k] = absum[o, k] = np.nan
            else:
                exact[o, k] = math.fsum(sel)
                absum[o, k] = math.fsum(np.abs(sel))
    return exact.reshape(kshape + (nbins,)), absum.reshape(kshape + (nbins,))


def depth(nslab, sms, P=1):
    """A bound on the roundings of any one value (DESIGN §3n): the lane-order group sum (31), the
    warp's run of steps over its split (at most nslab / 16 + 1: a warp step takes at least 4 slab
    items), the fold of the 4 warps (3), of the splits (at most 4 per SM) and of the P ranks."""
    return 31 + nslab // 16 + 1 + 3 + 4 * sms + P


def check(got, exact, absum, nslab, sms, single, P=1, what=""):
    eps = 2.0 ** -53
    tol = depth(nslab, sms, P) * eps * absum
    if single:
        tol = tol + np.abs(exact) * 2.0 ** -24
    got = got.astype(np.float64)
    assert got.shape == exact.shape, (what, got.shape, exact.shape)
    nan = np.isnan(exact)
    assert (np.isnan(got) == nan).all(), (what, np.argwhere(np.isnan(got) != nan)[:5])
    err = np.abs(got[~nan] - exact[~nan])
    assert (err <= tol[~nan] + 1e-300).all(), (what, err.max(), np.argwhere(err > tol[~nan])[:5])
