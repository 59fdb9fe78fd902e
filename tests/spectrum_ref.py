"""NumPy reference of shell-binned spectra (pa_shell_spectrum, DESIGN §3m) for the spectrum
tests: wavenumbers, Hermitian weights and bins elementwise in fp64 (each operation correctly
rounded, so bins match the library bit for bit), per-bin math.fsum of the contributions, per-bin
sum of |contribution| for the rounding bound, and the default bin count."""
import math

import numpy as np


def wavenumbers(n, r2c=False):
    """Integer wavenumbers of the global indices 0..n-1 (numpy's fftfreq order; r2c: the index)."""
    i = np.arange(n, dtype=np.int64)
    return i if r2c else np.where(i < (n + 1) // 2, i, i - n)


def weights(m, rfft_n):
    """Hermitian weights of the m bins of a real length rfft_n."""
    i = np.arange(m, dtype=np.int64)
    w = np.full(m, 2.0)
    w[i == 0] = 1.0
    if rfft_n % 2 == 0:
        w[i == rfft_n // 2] = 1.0
    return w


def default_rfft_n(size, rfft_dim):
    return max(0, 2 * (size[rfft_dim - 1] - 1)) if rfft_dim else 0


def shells(size, rfft_dim=None, scales=None, width=1.0):
    """floor(sqrt(q) / width + 0.5) of every mode, an fp64 array of `size` in logical order."""
    N = len(size)
    scales = scales or (1.0,) * N
    q = np.zeros(size)
    for d in range(N):
        k = scales[d] * wavenumbers(size[d], rfft_dim == d + 1).astype(np.float64)
        sh = [1] * N
        sh[d] = size[d]
        q = q + (k * k).reshape(sh)
    return np.floor(np.sqrt(q) / width + 0.5)


def mode_weights(size, rfft_dim=None, rfft_n=None):
    N = len(size)
    w = np.ones(size)
    if rfft_dim:
        n = default_rfft_n(size, rfft_dim) if rfft_n is None else rfft_n
        sh = [1] * N
        sh[rfft_dim - 1] = size[rfft_dim - 1]
        w = w * weights(size[rfft_dim - 1], n).reshape(sh)
    return w


def default_nbins(size, rfft_dim=None, scales=None, width=1.0):
    N = len(size)
    scales = scales or (1.0,) * N
    q = 0.0
    for d in range(N):
        top = 0 if size[d] == 0 else size[d] - 1 if rfft_dim == d + 1 else size[d] // 2
        k = scales[d] * float(top)
        q = q + k * k
    return int(math.floor(math.sqrt(q) / width + 0.5)) + 1


def contributions(x, y=None):
    """abs2(x) (or real(x * conj(y))) as the library computes it: in the element's precision,
    then in fp64."""
    y = x if y is None else y
    return (x.real * y.real + x.imag * y.imag).astype(np.float64)


def spectrum(x, N, nbins, y=None, rfft_dim=None, rfft_n=None, scales=None, width=1.0):
    """(exact, abs_sum) per bin (NaN: the bin holds a NaN): x (and y) in logical order, the N
    spatial dims first, extra dims last."""
    size = x.shape[:N]
    b = shells(size, rfft_dim, scales, width)
    w = mode_weights(size, rfft_dim, rfft_n)
    c = contributions(x, y) * w.reshape(size + (1,) * (x.ndim - N))
    bb = np.broadcast_to(b.reshape(size + (1,) * (x.ndim - N)), x.shape).reshape(-1)
    c = c.reshape(-1)
    exact = np.zeros(nbins)
    absum = np.zeros(nbins)
    for k in range(nbins):
        sel = c[bb == k]
        exact[k] = math.fsum(sel) if not np.isnan(sel).any() else np.nan
        absum[k] = math.fsum(np.abs(sel)) if not np.isnan(sel).any() else np.nan
    return exact, absum


def depth(n_local, sms, P=1):
    """A bound on the roundings of any one bin (DESIGN §3m): the lane-order group sum (31), the
    warp's run of steps (n / 128 + 4 V + 2), the fold of the 4 warps (3), of the CTAs (at most
    4 per SM) and of the P ranks."""
    return 31 + n_local // 128 + 12 + 3 + 4 * sms + P


def check_bins(got, exact, absum, n_local, sms, single, P=1, what=""):
    eps = 2.0 ** -53
    tol = depth(n_local, sms, P) * eps * absum
    if single:
        tol = tol + np.abs(exact) * 2.0 ** -24
    got = got.astype(np.float64)
    nan = np.isnan(exact)
    assert (np.isnan(got) == nan).all(), (what, np.flatnonzero(np.isnan(got) != nan)[:5])
    err = np.abs(got[~nan] - exact[~nan])
    assert (err <= tol[~nan] + 1e-300).all(), (what, err.max(), np.flatnonzero(err > tol[~nan])[:5])
