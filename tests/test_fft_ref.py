"""Self-tests of the extended-precision reference (tests/fft_ref.py), and the accuracy of the CPU
build of the FFT core (tests/fft_host_check.cpp, tests/rfft_host_check.cpp) measured against it
-- the yardstick for the GPU numbers in DESIGN.md §3b / §3c."""
import os
import subprocess

import numpy as np
import pytest

from fft_ref import (EPS, brfft_ld, extended_precision_available, fft_ld, line_errors, rfft_ld,
                     scaled_lines)

HERE = os.path.dirname(os.path.abspath(__file__))
LS = [1 << k for k in range(3, 11)]   # 8 ... 1024
NS = [1 << k for k in range(4, 12)]   # 16 ... 2048

pytestmark = pytest.mark.skipif(not extended_precision_available(),
                                reason="np.longdouble is not extended precision on this platform "
                                       "(eps >= 1e-18): the reference would be no better than a "
                                       "double-precision FFT")


def test_long_double_is_extended():
    assert np.finfo(np.longdouble).eps < 1e-18


@pytest.mark.parametrize("L", [8, 64, 256])
def test_against_mpmath_direct_dft(L):
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 40
    rng = np.random.default_rng(L)
    x = rng.standard_normal((2, L)) + 1j * rng.standard_normal((2, L))
    for sign in (-1, 1):
        got = fft_ld(x, sign)
        for j in range(x.shape[0]):
            xs = [mp.mpc(float(v.real), float(v.imag)) for v in x[j]]
            w = [mp.expjpi(mp.mpf(2 * sign * k) / L) for k in range(L)]
            ref = [mp.fsum(xs[n] * w[(n * k) % L] for n in range(L)) for k in range(L)]
            num = mp.sqrt(mp.fsum(abs(_mpc(mp, got[j, k]) - ref[k]) ** 2 for k in range(L)))
            den = mp.sqrt(mp.fsum(abs(r) ** 2 for r in ref))
            assert float(num / den) <= 1e-17, (L, sign, j, float(num / den))


def _mpc(mp, z):
    """long-double complex -> mpc (the shortest round-tripping decimal: within half an ulp)"""
    f = lambda v: mp.mpf(np.format_float_scientific(v, unique=True))  # noqa: E731
    return mp.mpc(f(np.real(z)), f(np.imag(z)))


@pytest.mark.parametrize("L", LS)
def test_fft_ld_against_numpy(L):
    rng = np.random.default_rng(L)
    x = scaled_lines(rng, 16, L)
    for sign in (-1, 1):
        ref = np.fft.fft(x) if sign < 0 else np.fft.ifft(x) * L
        mx, _ = line_errors(ref, fft_ld(x, sign))
        assert mx <= 2 * EPS * np.log2(L), (L, sign, mx)


@pytest.mark.parametrize("N", NS)
def test_rfft_ld_and_brfft_ld_against_numpy(N):
    rng = np.random.default_rng(N)
    x = scaled_lines(rng, 16, N, complex_=False)
    mx, _ = line_errors(np.fft.rfft(x), rfft_ld(x))
    assert mx <= 2 * EPS * np.log2(N)
    X = scaled_lines(rng, 16, N // 2 + 1)
    assert np.all(X[:, 0].imag != 0)
    mx, _ = line_errors(N * np.fft.irfft(X, n=N), brfft_ld(X, N))
    assert mx <= 2 * EPS * np.log2(N)


def test_line_errors_sees_a_wrong_small_line():
    ref = np.ones((3, 8)) * np.array([[1e10], [1.0], [1e-10]])
    got = ref.copy()
    got[2] = ref[1]   # the small line replaced by another line's values
    mx, rms = line_errors(got, ref)
    assert mx > 1e9 and rms > 1e8
    assert line_errors(ref, ref) == (0.0, 0.0)


# ---- the CPU build of the core: its per-line error is the yardstick of the GPU numbers ----
def _exe(tmp_path_factory, name):
    out = os.path.join(str(tmp_path_factory.mktemp(name)), name)
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(HERE, name + ".cpp")],
                   check=True)
    return out


@pytest.fixture(scope="module")
def fft_exe(tmp_path_factory):
    return _exe(tmp_path_factory, "fft_host_check")


@pytest.fixture(scope="module")
def rfft_exe(tmp_path_factory):
    return _exe(tmp_path_factory, "rfft_host_check")


def host_core_errors(fft_exe, L, sign, lines=8, logR1=0):
    rng = np.random.default_rng(100 + L)
    x = scaled_lines(rng, lines, L)
    args = [fft_exe, str(L), str(sign)] + ([str(logR1)] if logR1 else [])
    got = np.stack([np.frombuffer(subprocess.run(args, input=np.ascontiguousarray(l).tobytes(),
                                                 capture_output=True, check=True).stdout,
                                  dtype=np.complex128) for l in x])
    return line_errors(got, fft_ld(x, sign))


@pytest.mark.parametrize("L", LS)
def test_host_core_accuracy(fft_exe, L):
    """The core without FMA contraction: per-line error inside eps log2(L), with the kernel's
    radix-16 register first pass at L = 1024 and the radix-4 / 8 one of fft_lines = 4."""
    variants = [0] + ([4] if L == 1024 else []) + ([L.bit_length() - 1 - 6] if L in (256, 512) else [])
    for logR1 in variants:
        for sign in (-1, 1):
            mx, rms = host_core_errors(fft_exe, L, sign, logR1=logR1)
            assert mx <= EPS * np.log2(L), (L, sign, logR1, mx)


@pytest.mark.parametrize("N", NS)
def test_host_real_core_accuracy(rfft_exe, N):
    rng = np.random.default_rng(200 + N)
    x = scaled_lines(rng, 8, N, complex_=False)
    got = np.stack([np.frombuffer(subprocess.run([rfft_exe, str(N), "-1"], input=l.tobytes(),
                                                 capture_output=True, check=True).stdout,
                                  dtype=np.complex128) for l in x])
    mx, _ = line_errors(got, rfft_ld(x))
    assert mx <= EPS * np.log2(N), (N, "r2c", mx)
    X = scaled_lines(rng, 8, N // 2 + 1)
    got = np.stack([np.frombuffer(subprocess.run([rfft_exe, str(N), "1"], input=np.ascontiguousarray(l).tobytes(),
                                                 capture_output=True, check=True).stdout,
                                  dtype=np.float64) for l in X])
    mx, _ = line_errors(got, brfft_ld(X, N))
    assert mx <= EPS * np.log2(N), (N, "c2r", mx)
