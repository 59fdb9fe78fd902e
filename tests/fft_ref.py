"""Extended-precision reference transforms for the FFT kernels' tests.

`fft_ld` is a plain iterative radix-2 FFT over the last axis in `np.longdouble` (x86: 64-bit
mantissa, eps 1.1e-19), with twiddles cos / sin(2 pi k / L) evaluated in long double from a
long-double pi.  Its error is some 100x below a double-precision FFT's, so the error of a
kernel measured against it is the kernel's own.  The inputs are float64 (the kernels' inputs,
bit for bit); only the arithmetic is extended.

    fft_ld(x, sign)     sum_n x[n] exp(sign 2 pi i n k / L)      (unnormalised both ways)
    rfft_ld(x)          numpy.fft.rfft
    brfft_ld(X, N)      N * numpy.fft.irfft(X, n=N): bins 0 and N/2 lose their imaginary parts
    line_errors(got, ref) -> (max, rms) over the lines of ||got - ref||_2 / ||ref||_2
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble
CLD = np.clongdouble
PI_LD = LD("3.14159265358979323846264338327950288419716939937510")
EPS = np.finfo(np.float64).eps


def extended_precision_available() -> bool:
    return np.finfo(LD).eps < 1e-18


def _twiddles(L: int, sign: int) -> np.ndarray:
    k = np.arange(L // 2, dtype=LD)
    a = LD(2) * PI_LD * k / LD(L)
    return (np.cos(a) + LD(sign) * 1j * np.sin(a)).astype(CLD)


def _bitrev(L: int) -> np.ndarray:
    bits = L.bit_length() - 1
    r = np.zeros(L, dtype=np.int64)
    for b in range(bits):
        r |= ((np.arange(L) >> b) & 1) << (bits - 1 - b)
    return r


def fft_ld(x, sign: int = -1) -> np.ndarray:
    """Unnormalised DFT over the last axis in long double (decimation in time, radix 2)."""
    x = np.asarray(x)
    L = x.shape[-1]
    assert L >= 1 and L & (L - 1) == 0, L
    a = x.astype(CLD)[..., _bitrev(L)]
    w = _twiddles(L, sign)
    m = 1
    while m < L:
        # butterflies of span 2m: a[j] +- W_{2m}^j a[j+m], W_{2m}^j = w[j * L / (2m)]
        a = a.reshape(x.shape[:-1] + (L // (2 * m), 2, m))
        t = a[..., 1, :] * w[:: L // (2 * m)][:m]
        a = np.stack((a[..., 0, :] + t, a[..., 0, :] - t), axis=-2)
        m *= 2
    return a.reshape(x.shape)


def rfft_ld(x) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    N = x.shape[-1]
    return fft_ld(x.astype(LD), -1)[..., : N // 2 + 1]


def brfft_ld(X, N: int) -> np.ndarray:
    X = np.asarray(X).astype(CLD)
    assert X.shape[-1] == N // 2 + 1
    X[..., 0] = X[..., 0].real
    X[..., N // 2] = X[..., N // 2].real
    full = np.concatenate((X, np.conj(X[..., 1: N // 2][..., ::-1])), axis=-1)
    return fft_ld(full, +1).real


def line_errors(got, ref):
    """(max, rms) over lines (last axis) of the relative 2-norm error; lines whose reference is
    exactly zero must be exactly zero too (their error counts as inf otherwise)."""
    got = np.asarray(got).astype(CLD if np.iscomplexobj(got) or np.iscomplexobj(ref) else LD)
    ref = np.asarray(ref)
    d = np.sqrt(np.sum(np.abs(got - ref) ** 2, axis=-1))
    n = np.sqrt(np.sum(np.abs(ref) ** 2, axis=-1))
    e = np.where(n > 0, d / np.where(n > 0, n, 1), np.where(d > 0, np.inf, 0))
    e = np.asarray(e, dtype=np.float64).reshape(-1)
    return float(e.max()), float(np.sqrt(np.mean(e ** 2)))


def scaled_lines(rng, nlines: int, L: int, complex_: bool = True, smin: int = -40, smax: int = 40):
    """`nlines` random lines, line j scaled by 2^s with s cycling over smin..smax: the scaling is
    exact, so the reference stays exact, and a value read from the wrong line shows up as a
    per-line error of order 2^|s1 - s2|."""
    shape = (nlines, L)
    x = rng.standard_normal(shape) + (1j * rng.standard_normal(shape) if complex_ else 0)
    s = np.array([smin + (j * 7) % (smax - smin + 1) for j in range(nlines)], dtype=np.float64)
    return x * np.exp2(s)[:, None]
